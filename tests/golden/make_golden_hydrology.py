"""Golden vectors for river routing, produced by the reference's own `d8_flow`, `flow_accumulation` and
`plot_flow_indicator` (terrain_diffusion/inference/postprocessing.py).  That module imports matplotlib and torch at the
top, so the functions are extracted from its source with `ast` and run with numpy (and heapq) alone.  Only outputs
are stored (tests/golden/hydrology_golden.npz): per case `<name>.kmax` (int8), `<name>.is_sink`, `<name>.A` (fp32) and
`<name>.ind<k>` for each pool kernel k; inputs are regenerated from seeds by tests/_hydrology_inputs.py.  The
FILLED_CASES are routed after the reference's `fill_depressions_priority_flood`, whose result is stored as
`<name>.filled`.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_hydrology.py
"""
from __future__ import annotations

import ast
import heapq
import os
import sys
import warnings
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])
sys.path[:0] = [str(ROOT)]

from tests._hydrology_inputs import CASES, FILLED_CASES, hydrology_case  # noqa: E402

NAMES = ("d8_flow", "flow_accumulation", "plot_flow_indicator", "fill_depressions_priority_flood")


def reference_functions():
    src = (REF / "terrain_diffusion/inference/postprocessing.py").read_text()
    body = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in NAMES]
    assert len(body) == len(NAMES), "d8_flow / flow_accumulation / plot_flow_indicator / the fill not found"
    ns = {"np": np, "heapq": heapq}
    exec(compile(ast.Module(body=body, type_ignores=[]), "postprocessing_extract", "exec", dont_inherit=True), ns)
    return [ns[n] for n in NAMES]


def main():
    d8_flow, flow_accumulation, plot_flow_indicator, fill = reference_functions()
    out = {}
    cases = [(name, *hydrology_case(name)) for name in CASES]
    for name, (build, pools) in FILLED_CASES.items():
        out[f"{name}.filled"] = filled = fill(build())
        assert filled.dtype == np.float32
        cases.append((name, filled, 1e-3, pools))
    for name, z, tol, pools in cases:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)      # NaN arithmetic in the slope stack
            rr, cc, is_sink, kmax = d8_flow(z, tol=tol)
            a = flow_accumulation(z, rr, cc, is_sink)
            inds = {k: plot_flow_indicator(z, max_pool_kernel=k) for k in pools}
        assert kmax.min() >= 0 and kmax.max() < 8 and a.dtype == np.float32
        out[f"{name}.kmax"] = kmax.astype(np.int8)
        out[f"{name}.is_sink"] = is_sink
        out[f"{name}.A"] = a
        for k, ind in inds.items():
            assert ind.dtype == np.float32
            out[f"{name}.ind{k}"] = ind
        print(name, z.shape, "tol", tol, "sinks", int(is_sink.sum()), "max A", float(a.max()),
              {k: v.shape for k, v in inds.items()})
    np.savez_compressed(HERE / "hydrology_golden.npz", **out)
    print("wrote", HERE / "hydrology_golden.npz", (HERE / "hydrology_golden.npz").stat().st_size // 1024, "KiB")


if __name__ == "__main__":
    main()
