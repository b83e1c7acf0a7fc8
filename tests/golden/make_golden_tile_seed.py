"""Golden tile seeds at large tile indices, produced by the reference's own `_tile_seed`
(terrain_diffusion/inference/world_pipeline.py), which masks each index to 32 bits.  That module imports torch and the
models at the top, so the function is extracted from its source with `ast`.  Writes tests/golden/tile_seed_golden.npz:
`tile_seed_large.base` (uint64), `tile_seed_large.args` (int64 [n, 2]: ty, tx) and `tile_seed_large.out` (uint64).

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_tile_seed.py
"""
from __future__ import annotations

import ast
import os
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])

BASES = (0, 1, 12345, 2 ** 63 + 11, 2 ** 64 - 1)
INDICES = (0, -1, 2 ** 31 - 1, 2 ** 31, -2 ** 31, -2 ** 31 - 1, 2 ** 32, -2 ** 32, 2 ** 32 + 7, 5 * 2 ** 32 + 3,
           -3 * 2 ** 32 - 9, 2 ** 62, -2 ** 63, 2 ** 63 - 1)


def main():
    src = (REF / "terrain_diffusion/inference/world_pipeline.py").read_text()
    body = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "_tile_seed"]
    assert len(body) == 1, "_tile_seed not found"
    ns: dict = {}
    exec(compile(ast.Module(body=body, type_ignores=[]), "world_pipeline_extract", "exec", dont_inherit=True), ns)
    bases, args, outs = [], [], []
    for i, b in enumerate(BASES):
        for j, ty in enumerate(INDICES):
            tx = INDICES[(i + 3 * j) % len(INDICES)]
            bases.append(b)
            args.append((ty, tx))
            outs.append(ns["_tile_seed"](b, ty, tx))
    np.savez_compressed(HERE / "tile_seed_golden.npz", **{
        "tile_seed_large.base": np.array(bases, np.uint64), "tile_seed_large.args": np.array(args, np.int64),
        "tile_seed_large.out": np.array(outs, np.uint64)})
    print("wrote", len(outs), "tile seeds to", HERE / "tile_seed_golden.npz")


if __name__ == "__main__":
    main()
