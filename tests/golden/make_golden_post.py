"""Golden vectors for the elevation read-out (SURVEY.md section 8(f) rank 3), produced by the reference's own code:
`terrain_diffusion/data/laplacian_encoder.py` is imported unchanged (it needs only torch + torchvision, both present in
this container) and `WorldPipeline._compute_elev` is extracted from the reference source with `ast` and called with a
stand-in `self` (world_pipeline.py itself cannot be imported: infinite_tensor, h5py, rasterio ... are absent).
Only outputs are stored (tests/golden/post_golden.npz, and the coastal climate case in post_coastal_golden.npz); inputs
are regenerated from seeds by tests/_post_inputs.py.

    python tests/golden/make_golden_post.py            # both files
    python tests/golden/make_golden_post.py coastal    # post_coastal_golden.npz only
"""
from __future__ import annotations

import os

import ast
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]

from terrain_diffusion.data.laplacian_encoder import laplacian_decode, laplacian_denoise  # noqa: E402

from tests._post_inputs import (COASTAL_SCALE, COASTAL_WINDOW, ELEV_WINDOWS, RESIDUAL_MEAN, RESIDUAL_STD,  # noqa: E402
                                coarse_canvas, coastal_canvas, coastal_elev, elev_canvases, laplacian_case)

torch.set_grad_enabled(False)


class TorchCanvas:
    def __init__(self, fake):
        self.fake = fake

    def __getitem__(self, key):
        _, ys, xs = key
        return torch.from_numpy(self.fake.planes(ys.start, ys.stop, xs.start, xs.stop).copy())


def extract():
    """WorldPipeline._compute_elev / _compute_climate and local_baseline_temperature_torch as plain functions."""
    src = (REF / "terrain_diffusion/inference/world_pipeline.py").read_text()
    tree = ast.parse(src)
    body = []
    for n in tree.body:
        if isinstance(n, ast.ClassDef) and n.name == "WorldPipeline":
            body += [m for m in n.body if isinstance(m, ast.FunctionDef) and m.name in ("_compute_elev", "_compute_climate")]
    assert len(body) == 2, "WorldPipeline._compute_elev / _compute_climate not found"
    # local_baseline_temperature_torch lives in inference/postprocessing.py, which imports matplotlib (absent here):
    # the function definition alone is extracted the same way
    pp = ast.parse((REF / "terrain_diffusion/inference/postprocessing.py").read_text())
    body += [n for n in pp.body if isinstance(n, ast.FunctionDef) and n.name == "local_baseline_temperature_torch"]
    assert len(body) == 3
    import torch.nn.functional as F
    ns = {"torch": torch, "np": np, "F": F, "laplacian_denoise": laplacian_denoise, "laplacian_decode": laplacian_decode}
    exec(compile(ast.Module(body=body, type_ignores=[]), "world_pipeline_extract", "exec"), ns)
    return ns


def main(ns):
    out = {}
    for name in ("rect", "square", "wide"):
        r, l = laplacian_case(name)
        r_t, l_t = torch.from_numpy(r), torch.from_numpy(l)
        r2, l2 = laplacian_denoise(r_t, l_t, sigma=5)
        out[f"lap_{name}_lowres"] = l2.numpy()
        out[f"lap_{name}_elev"] = laplacian_decode(r2, l2).numpy()
        out[f"lap_{name}_decode_extrap"] = laplacian_decode(r_t, l_t, extrapolate=True).numpy()
    resid, lat = elev_canvases()
    fake = SimpleNamespace(kwargs={"residual_mean": RESIDUAL_MEAN, "residual_std": RESIDUAL_STD}, latents=TorchCanvas(lat),
                           coarse=TorchCanvas(coarse_canvas()))
    for name, (i1, j1, i2, j2) in ELEV_WINDOWS.items():
        elev = ns["_compute_elev"](fake, i1, j1, i2, j2, TorchCanvas(resid), 8)
        out[f"elev_{name}"] = elev.numpy()
        clim = ns["_compute_climate"](fake, i1, j1, i2, j2, elev, 8)
        out[f"climate_{name}"] = clim.numpy()[:, ::2, ::2]        # every other pixel: keeps the fixture small
        print(name, tuple(elev.shape), float(elev.abs().max()), tuple(clim.shape), [round(float(c.mean()), 4) for c in clim])
    np.savez_compressed(HERE / "post_golden.npz", **out)
    print("wrote", HERE / "post_golden.npz", sum(v.nbytes for v in out.values()) // 1024, "KiB raw")


def coastal(ns):
    """The coastal climate case (tests/_post_inputs.coastal_canvas) in a file of its own, so post_golden.npz stays as
    recorded: the reference's local_baseline_temperature_torch on the normalised coarse map compute_climate builds, and
    its _compute_climate over COASTAL_WINDOW (stored at every fourth pixel)."""
    i1, j1, i2, j2 = COASTAL_WINDOW
    cc = coastal_canvas()
    fake = SimpleNamespace(coarse=TorchCanvas(cc))
    S = 32 * COASTAL_SCALE
    ci1, cj1, ci2, cj2 = i1 // S, j1 // S, -((-i2) // S), -((-j2) // S)
    c = torch.from_numpy(cc.planes(ci1 - 8, ci2 + 8, cj1 - 8, cj2 + 8).copy())
    cmap = c[:-1] / c[-1:]
    e = torch.sign(cmap[0]) * torch.square(torch.maximum(torch.zeros_like(cmap[0]), cmap[0]))
    t_sea, beta = ns["local_baseline_temperature_torch"](cmap[2], e, win=15, fallback_threshold=0.02)
    clim = ns["_compute_climate"](fake, i1, j1, i2, j2, torch.from_numpy(coastal_elev()), COASTAL_SCALE)
    out = {"t_sea": t_sea[0].numpy(), "beta": beta[0].numpy(), "climate": clim.numpy()[:, ::4, ::4]}
    np.savez_compressed(HERE / "post_coastal_golden.npz", **out)
    print("wrote", HERE / "post_coastal_golden.npz", sum(v.nbytes for v in out.values()) // 1024, "KiB raw")


if __name__ == "__main__":
    extracted = extract()
    if sys.argv[1:] != ["coastal"]:
        main(extracted)
    coastal(extracted)
