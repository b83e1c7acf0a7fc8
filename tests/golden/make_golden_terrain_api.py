"""Golden vectors for the terrain API read-out, produced by the reference's own `_get_terrain`, `_binary_response` and
`_elev_to_int16` (terrain_diffusion/inference/api.py:73-166).  That module imports flask and click and builds a
WorldPipeline, so the three functions are extracted from its source with `ast` and run with torch, numpy, a stand-in
`Response` that records the body and headers, and the analytic world of tests/_terrain_api_inputs.py (whose `get()`
returns slices of a seeded field on absolute coordinates).  Stored per case: the fp32 elevation and climate `_get_terrain`
returns, and the response body and its X-Height / X-Width headers.  The file also records torch's version and its CPU
dispatch capability: torch picks its bilinear kernels (and so their rounding) per build and per CPU.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_terrain_api.py
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

from tests._terrain_api_inputs import CASES, case_world  # noqa: E402

NAMES = ("_elev_to_int16", "_binary_response", "_get_terrain")


class Response:
    """flask.Response as _binary_response uses it: the body and a headers mapping."""

    def __init__(self, payload, mimetype=None):
        self.body, self.mimetype, self.headers = bytes(payload), mimetype, {}


def reference_api():
    src = (REF / "terrain_diffusion/inference/api.py").read_text()
    body = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in NAMES]
    assert len(body) == len(NAMES), "api.py functions not found"
    code = compile(ast.Module(body=body, type_ignores=[]), "api_extract", "exec", dont_inherit=True)
    ns = {"np": np, "torch": torch, "Response": Response, "Optional": Optional, "Tuple": Tuple,
          "WorldPipeline": object}
    exec(code, ns)
    return {n: ns[n] for n in NAMES}


def reference_terrain(api, world, i1, j1, i2, j2, scale):
    """What GET /terrain computes after argument parsing (api.py:200-201)."""
    out = api["_get_terrain"](world, i1, j1, i2, j2, scale)
    resp = api["_binary_response"](out["elev"], out.get("climate"))
    return out, resp


def main():
    api = reference_api()
    store = {"torch_version": np.array(torch.__version__),
             "cpu_capability": np.array(torch.backends.cpu.get_cpu_capability())}
    for name in CASES:
        world, (i1, j1, i2, j2, scale) = case_world(name)
        out, resp = reference_terrain(api, world, i1, j1, i2, j2, scale)
        elev, clim = out["elev"].numpy(), out["climate"].numpy()
        assert elev.shape == (i2 - i1, j2 - j1) and clim.shape == (5, i2 - i1, j2 - j1)
        store[f"{name}.elev"] = np.ascontiguousarray(elev)
        store[f"{name}.climate"] = np.ascontiguousarray(clim)
        store[f"{name}.body"] = np.frombuffer(resp.body, np.uint8)
        store[f"{name}.hw"] = np.array([int(resp.headers["X-Height"]), int(resp.headers["X-Width"])])
        print(name, elev.shape, "native", world.calls[-1], "NaN elev", int(np.isnan(elev).sum()), "body", len(resp.body))
    np.savez_compressed(HERE / "terrain_api_golden.npz", **store)
    print("wrote", HERE / "terrain_api_golden.npz", "torch", torch.__version__,
          torch.backends.cpu.get_cpu_capability())


if __name__ == "__main__":
    main()
