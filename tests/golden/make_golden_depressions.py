"""Golden vectors for depression filling and river-bed smoothing, produced by the reference's own
`fill_depressions_priority_flood` and `smooth_river_bumps` (terrain_diffusion/inference/postprocessing.py), and for
the routing of a filled window through its `d8_flow`, `flow_accumulation` and `plot_flow_indicator`.  That module
imports matplotlib and torch at the top, so the functions are extracted from its source with `ast` and run with
numpy and heapq alone.  Only outputs are stored (tests/golden/depressions_golden.npz): `fill.<name>` and
`smooth.<name>` (fp32) per case, and `compose.filled`, `compose.A`, `compose.ind1`; inputs are regenerated from seeds
by tests/_depression_inputs.py.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_depressions.py
"""
from __future__ import annotations

import ast
import heapq
import os
import sys
import time
import warnings
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])
sys.path[:0] = [str(ROOT)]

from tests._depression_inputs import FILL_CASES, SMOOTH_CASES, composition_case, fill_case, smooth_case  # noqa: E402

NAMES = ("d8_flow", "flow_accumulation", "plot_flow_indicator", "smooth_river_bumps",
         "fill_depressions_priority_flood")


def reference_functions():
    src = (REF / "terrain_diffusion/inference/postprocessing.py").read_text()
    body = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in NAMES]
    assert len(body) == len(NAMES), "a river function of postprocessing.py was not found"
    ns = {"np": np, "heapq": heapq}
    exec(compile(ast.Module(body=body, type_ignores=[]), "postprocessing_extract", "exec", dont_inherit=True), ns)
    return [ns[n] for n in NAMES]


def main():
    d8_flow, flow_accumulation, plot_flow_indicator, smooth, fill = reference_functions()
    out = {}
    for name in FILL_CASES:
        z, kw = fill_case(name)
        t0 = time.perf_counter()
        f = fill(z, **kw)
        assert f.dtype == np.float32 and f.shape == z.shape
        out[f"fill.{name}"] = f
        print("fill", name, z.shape, kw, "raised", int((f > z).sum()), f"{time.perf_counter() - t0:.2f} s")
    for name in SMOOTH_CASES:
        z, kw = smooth_case(name)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            s = smooth(z, **kw)
        assert s.dtype == np.float32 and s.shape == z.shape
        out[f"smooth.{name}"] = s
        print("smooth", name, z.shape, kw)
    z = composition_case()
    filled = fill(z)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)      # NaN arithmetic in the slope stack
        rr, cc, is_sink, _ = d8_flow(filled)
        out["compose.A"] = flow_accumulation(filled, rr, cc, is_sink)
        out["compose.ind1"] = plot_flow_indicator(filled)
    out["compose.filled"] = filled
    print("compose: land sinks", int((is_sink & ~(np.isnan(filled) | (filled <= 0))).sum()),
          "max A", float(out["compose.A"].max()))
    np.savez_compressed(HERE / "depressions_golden.npz", **out)
    print("wrote", HERE / "depressions_golden.npz", (HERE / "depressions_golden.npz").stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
