"""Golden vectors for the shaded relief map, produced by the reference's own `get_relief_map`
(terrain_diffusion/inference/relief_map.py).  That module imports matplotlib, which is absent here, so `_to_numpy` and
`get_relief_map` are extracted from its source with `ast`, compiled with the `annotations` future flag the file carries,
and run with numpy, scipy's `gaussian_filter` and a stand-in `plt` whose `get_cmap("terrain")` is the restated
colormap (oracle/relief.py `terrain_cmap`).  Only outputs are stored (tests/golden/relief_golden.npz), every other row
and column of the cases larger than 64 x 64 (tests/_relief_inputs.py `golden_stride`); inputs are regenerated from
seeds by tests/_relief_inputs.py.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_relief.py
"""
from __future__ import annotations

import __future__
import ast
import os
import sys
import warnings
from pathlib import Path
from types import SimpleNamespace

import numpy as np
from scipy.ndimage import gaussian_filter

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])
sys.path[:0] = [str(ROOT)]

from oracle.relief import terrain_cmap  # noqa: E402
from tests._relief_inputs import CASES, golden_stride, relief_case  # noqa: E402


def reference_get_relief_map():
    src = (REF / "terrain_diffusion/inference/relief_map.py").read_text()
    body = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in ("_to_numpy", "get_relief_map")]
    assert len(body) == 2, "_to_numpy / get_relief_map not found"
    code = compile(ast.Module(body=body, type_ignores=[]), "relief_map_extract", "exec",
                   flags=__future__.annotations.compiler_flag, dont_inherit=True)
    plt = SimpleNamespace(get_cmap=lambda name: terrain_cmap if name == "terrain" else None)
    ns = {"np": np, "gaussian_filter": gaussian_filter, "plt": plt}
    exec(code, ns)
    return ns["get_relief_map"]


def main():
    ref = reference_get_relief_map()
    out = {}
    for name in CASES:
        elev, kw = relief_case(name)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)       # negative norm ** 0.7 in the vrange case
            rgb = ref(elev, None, None, None, **kw)
        assert rgb.dtype == np.float32 and rgb.shape == elev.shape + (3,)
        s = golden_stride(name)
        out[name] = np.ascontiguousarray(rgb[::s, ::s])
        print(name, elev.shape, kw, "NaN px", int(np.isnan(rgb[..., 0]).sum()), "mean", np.nanmean(rgb, axis=(0, 1)))
    np.savez_compressed(HERE / "relief_golden.npz", **out)
    print("wrote", HERE / "relief_golden.npz", sum(v.nbytes for v in out.values()) // 1024, "KiB raw")


if __name__ == "__main__":
    main()
