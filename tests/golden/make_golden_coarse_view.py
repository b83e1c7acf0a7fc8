"""Golden vectors for the explorer's coarse map and the random sampler's land search, produced by the reference's own
functions: `_coarse_channel`, `_png_response`, `coarse_png`, `coarse_data` and `coarse_stats`
(terrain_diffusion/inference/explorer/server.py), `sample_land_tiles` and `get_coarse_climate_info`
(inference/random_sampler.py) and `normalize_tensor` (inference/world_pipeline.py).  Their modules import flask,
matplotlib, PIL and click, which are absent here, so the functions are extracted from the source with `ast` (route
decorators dropped) and run with stand-ins:

* `request.args`: Flask's `args.get(key, default, type)` over the case's arguments;
* `_get_pipeline()` / the sampler's `world`: a world whose `coarse[:, ci0:ci1, cj0:cj1]` returns the seeded analytic
  sums of tests/_coarse_view_inputs.py on absolute cell coordinates as a CPU tensor;
* `Response`, `jsonify` (which raises in the png / stats handlers' error branch, so an error cannot pass for a result,
  and returns its payload for `coarse_data`'s success) and `plt.imsave` from tests/golden/make_golden_explorer.py, with
  its restated matplotlib 3.9 `Normalize`, `Colormap` and `to_rgba(bytes=True)`;
* `plt.get_cmap('viridis')`: that `Colormap` over the seeded 256-entry table of tests/_coarse_view_inputs.py, so the
  handler logic is pinned independently of viridis' values.

Stored (tests/golden/coarse_view_golden.npz): per png case the uint8 RGBA, vmin / vmax and the two headers; per data
case the rounded channels; per stats case the min / max; per land case the tile list; per sample case the pick after
random.seed(seed); per climate cell the four values; the table and the numpy version.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_coarse_view.py
"""
from __future__ import annotations

import __future__
import ast
import io
import random
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path[:0] = [str(ROOT)]

from tests._coarse_view_inputs import (CLIMATE_CELLS, DATA_CASES, LAND_CASES, PNG_CASES, SAMPLE_CASES,  # noqa: E402
                                       seeded_lut, world_sums)
from tests.golden.make_golden_explorer import (REF, Args, Colormap, Normalize, Response,  # noqa: E402
                                               to_rgba_bytes)


class FakeCoarse:
    def __init__(self, kind):
        self.kind, self.reads = kind, []

    def __getitem__(self, key):
        _, ys, xs = key
        self.reads.append((ys.start, ys.stop, xs.start, xs.stop))
        return torch.from_numpy(world_sums(self.kind, ys.start, ys.stop, xs.start, xs.stop))


def extract(path, names):
    tree = ast.parse((REF / path).read_text())
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in body) == sorted(names), f"{names} not all found in {path}"
    for n in body:
        n.decorator_list = []
    return compile(ast.Module(body=body, type_ignores=[]), str(path), "exec",
                   flags=__future__.annotations.compiler_flag, dont_inherit=True)


def reference_functions():
    state = SimpleNamespace(world=None, images=[])

    def imsave(fname, arr, format=None):
        state.images.append(to_rgba_bytes(arr))
        fname.write(b"PNG stand-in")

    def jsonify(payload):
        if isinstance(payload, dict) and "error" in payload:
            raise RuntimeError(f"the handler failed: {payload}")
        return payload

    table = seeded_lut()
    ns = {"io": io, "np": np, "torch": torch, "random": random, "Response": Response, "jsonify": jsonify,
          "CHANNEL_NAMES": ["Elev", "p5", "Temp", "T std", "Precip", "Precip CV"],
          "matplotlib": SimpleNamespace(colors=SimpleNamespace(Normalize=Normalize)),
          "plt": SimpleNamespace(get_cmap={"viridis": Colormap(table)}.__getitem__, imsave=imsave),
          "request": SimpleNamespace(args=None), "_get_pipeline": lambda: state.world}
    exec(extract("terrain_diffusion/inference/world_pipeline.py", ["normalize_tensor"]), ns)
    exec(extract("terrain_diffusion/inference/explorer/server.py",
                 ["_coarse_channel", "_png_response", "coarse_png", "coarse_data", "coarse_stats"]), ns)
    exec(extract("terrain_diffusion/inference/random_sampler.py", ["sample_land_tiles", "get_coarse_climate_info"]),
         ns)

    def run(name, world, args):
        state.world, state.images = world, []
        ns["request"].args = Args(args)
        return ns[name](), state

    return run, ns, table


def main():
    run, ns, table = reference_functions()
    out = {"numpy_version": np.array(np.__version__), "lut": table}
    for name, (kind, args) in PNG_CASES.items():
        world = SimpleNamespace(coarse=FakeCoarse(kind))
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            resp, state = run("coarse_png", world, args)
        assert isinstance(resp, Response) and resp.mimetype == "image/png" and len(state.images) == 1, resp
        out[f"png.{name}.image"] = state.images[0]
        out[f"png.{name}.headers"] = np.array([resp.headers["X-Vmin"], resp.headers["X-Vmax"]])
        print("png", name, state.images[0].shape, resp.headers["X-Vmin"], resp.headers["X-Vmax"],
              "reads", len(world.coarse.reads), "opaque", int((state.images[0][..., 3] == 255).sum()))
    for name, (kind, args) in DATA_CASES.items():
        world = SimpleNamespace(coarse=FakeCoarse(kind))
        with np.errstate(invalid="ignore", divide="ignore"):
            data, _ = run("coarse_data", world, args)
            stats, _ = run("coarse_stats", world, args)
        assert [data[k] for k in ("ci0", "ci1", "cj0", "cj1")] == [args[k] for k in ("ci0", "ci1", "cj0", "cj1")]
        out[f"data.{name}"] = np.array([data["channels"][n] for n in ns["CHANNEL_NAMES"]], np.float64)
        out[f"stats.{name}"] = np.array([[stats[c]["min"], stats[c]["max"]] for c in range(6)], np.float64)
        assert [stats[c]["name"] for c in range(6)] == ns["CHANNEL_NAMES"]
        print("data", name, out[f"data.{name}"].shape, "stats", out[f"stats.{name}"].tolist())
    world = SimpleNamespace(coarse=FakeCoarse("mixed"))
    for cw, detail, frac in LAND_CASES:
        # n_samples above any count: the reference returns valid_tiles itself, in its order
        tiles = ns["sample_land_tiles"](world, cw, detail, frac, n_samples=10 ** 9)
        out[f"land.{cw}.{detail}.{frac}"] = np.array(tiles, np.int64).reshape(-1, 2)
        print("land", cw, detail, frac, len(tiles))
    from tests._coarse_view_inputs import LAND_WINDOW
    for seed, detail, frac, n in SAMPLE_CASES:
        random.seed(seed)
        pick = ns["sample_land_tiles"](world, LAND_WINDOW, detail, frac, n)
        out[f"sample.{seed}"] = np.array(pick, np.int64).reshape(-1, 2)
        print("sample", seed, len(pick))
    nan_world = SimpleNamespace(coarse=FakeCoarse("nan"))
    for ci, cj in CLIMATE_CELLS:
        with np.errstate(invalid="ignore", divide="ignore"):
            info = ns["get_coarse_climate_info"](nan_world, ci, cj)
        assert sorted(info) == ["precip", "precip_cv", "temp", "temp_std"]
        out[f"climate.{ci}.{cj}"] = np.array([info["temp"], info["temp_std"], info["precip"], info["precip_cv"]])
        print("climate", ci, cj, out[f"climate.{ci}.{cj}"])
    np.savez_compressed(HERE / "coarse_view_golden.npz", **out)
    print("wrote", HERE / "coarse_view_golden.npz", "numpy", np.__version__)


if __name__ == "__main__":
    main()
