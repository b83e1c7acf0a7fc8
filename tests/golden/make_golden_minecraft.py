"""Golden vectors for the Minecraft API read-out, produced by the reference's own `_compute_climate_vars`,
`_get_upsampled`, `_classify_biome`, `_transform_to_int16_bytes` and `_binary_response`
(terrain_diffusion/inference/minecraft_api.py:83-688).  That module imports flask, click and pyfastnoiselite and builds
a WorldPipeline, so the five functions and the module-level `_BIOME_ID` and noise-generator assignments are extracted
from its source with `ast` and run with torch, numpy, a stand-in `Response`, the stand-in FastNoiseLite of
tests/_minecraft_inputs.py (also installed as `pyfastnoiselite.pyfastnoiselite`) and its analytic `BiomeWorld`.  Each case
runs the body of `_handle_1x` (:714-727) or `_handle_upsampled` (:730-745) after argument parsing.  Stored per case:
the X-Height / X-Width headers, a SHA-256 digest (tests/_minecraft_inputs.digest) of the response body and of the
elevation, smooth elevation, climate and biome ids, the body itself for windows of at most BODY_LIMIT pixels and the
arrays themselves for windows of at most FULL_LIMIT pixels; for a one-column window, the error the reference raises.  The file also records torch's version and CPU dispatch capability: torch picks its bilinear and conv2d kernels (and so their
rounding) per build and per CPU.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_minecraft.py
"""
from __future__ import annotations

import ast
import os
import sys
from pathlib import Path
from typing import Optional, Tuple

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])
sys.path[:0] = [str(ROOT)]

from tests._minecraft_inputs import BODY_LIMIT, CASES, FULL_LIMIT, case_world, digest, install_stand_in  # noqa: E402

NAMES = ("_transform_to_int16_bytes", "_binary_response", "_compute_climate_vars", "_get_upsampled", "_classify_biome")
GENERATORS = ("_TEMP_NOISE", "_TEMP_NOISE_FINE", "_PRECIP_NOISE", "_SNOW_NOISE", "_SNOW_NOISE_FINE",
              "_ELEV_NOISE_COARSE", "_ELEV_NOISE_FINE")


class Response:
    """flask.Response as _binary_response uses it: the body and a headers mapping."""

    def __init__(self, payload, mimetype=None):
        self.body, self.mimetype, self.headers = bytes(payload), mimetype, {}


def _assigns_module_name(node) -> bool:
    if not isinstance(node, ast.Assign) or len(node.targets) != 1:
        return False
    t = node.targets[0]
    if isinstance(t, ast.Name):
        return t.id == "_BIOME_ID" or t.id in GENERATORS
    return isinstance(t, ast.Attribute) and isinstance(t.value, ast.Name) and t.value.id in GENERATORS


def reference_module():
    src = (REF / "terrain_diffusion/inference/minecraft_api.py").read_text()
    tree = ast.parse(src)
    funcs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in NAMES]
    assert len(funcs) == len(NAMES), "minecraft_api.py functions not found"
    assigns = [n for n in tree.body if _assigns_module_name(n)]
    assert sum(isinstance(n.targets[0], ast.Name) for n in assigns) == len(GENERATORS) + 1
    code = compile(ast.Module(body=assigns + funcs, type_ignores=[]), "minecraft_api_extract", "exec",
                   dont_inherit=True)
    fnl = install_stand_in()
    ns = {"np": np, "torch": torch, "Response": Response, "Optional": Optional, "Tuple": Tuple,
          "WorldPipeline": object, "FastNoiseLite": fnl.FastNoiseLite, "NoiseType": fnl.NoiseType,
          "FractalType": fnl.FractalType}
    exec(code, ns)
    return ns


def handle(ref, world, i1, j1, i2, j2, scale, noise):
    """_handle_1x / _handle_upsampled after _parse_quad, _parse_noise and _maybe_update_seed, binary format."""
    if scale == 1:
        out_pad = world.get(i1 - 1, j1 - 1, i2 + 1, j2 + 1, with_climate=False)
        elev_padded = out_pad["elev"]
        out = world.get(i1, j1, i2, j2, with_climate=True)
        elev, climate = out["elev"], out.get("climate")
        biome = ref["_classify_biome"](elev, climate, i1, j1, elev_padded=elev_padded,
                                       pixel_size_m=world.native_resolution)
        return {"elev": elev, "elev_smooth": elev, "climate": climate, "biome": biome}, \
            ref["_binary_response"](elev, biome=biome)
    pixel_size_m = world.native_resolution / scale
    out = ref["_get_upsampled"](world, i1, j1, i2, j2, scale=scale, noise_scale=noise, pixel_size_m=pixel_size_m)
    biome = ref["_classify_biome"](out["elev_smooth"], out.get("climate"), i1, j1, elev_padded=out["elev_padded"],
                                   pixel_size_m=pixel_size_m)
    return {"elev": out["elev"], "elev_smooth": out["elev_smooth"], "climate": out["climate"], "biome": biome}, \
        ref["_binary_response"](out["elev"], biome=biome)


def main():
    ref = reference_module()
    store = {"torch_version": np.array(torch.__version__),
             "cpu_capability": np.array(torch.backends.cpu.get_cpu_capability())}
    for name in CASES:
        world, (i1, j1, i2, j2, scale, noise) = case_world(name)
        H, W = i2 - i1, j2 - j1
        try:
            out, resp = handle(ref, world, i1, j1, i2, j2, scale, noise)
        except IndexError as e:
            # A one-column window taller than one pixel: the reference's Sobel `.squeeze()` drops the column axis, its
            # [H] gradient broadcasts against [H, 1] masks to [H, H], and the first mask write raises.
            assert W == 1 and H > 1, (name, e)
            store[f"{name}.error"] = np.array(f"{type(e).__name__}: {e}")
            print(name, (H, W), "reference raises", store[f"{name}.error"])
            continue
        for k in ("elev", "elev_smooth", "climate", "biome"):
            v = out[k].numpy()
            assert v.shape[-2:] == (H, W), (name, k, v.shape)
            store[f"{name}.{k}.sha256"] = np.array(digest(v))
            if H * W <= FULL_LIMIT:
                store[f"{name}.{k}"] = np.ascontiguousarray(v)
        ids, counts = np.unique(out["biome"].numpy(), return_counts=True)
        body = np.frombuffer(resp.body, np.uint8)
        store[f"{name}.body.sha256"] = np.array(digest(body))
        if H * W <= BODY_LIMIT:
            store[f"{name}.body"] = body
        store[f"{name}.hw"] = np.array([int(resp.headers["X-Height"]), int(resp.headers["X-Width"])])
        print(name, (H, W), "reads", world.calls, "ids", dict(zip(ids.tolist(), counts.tolist())))
    np.savez_compressed(HERE / "minecraft_golden.npz", **store)
    print("wrote", HERE / "minecraft_golden.npz", "torch", torch.__version__,
          torch.backends.cpu.get_cpu_capability())


if __name__ == "__main__":
    main()
