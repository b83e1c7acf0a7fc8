"""Golden vectors for the coarse stage's synthetic conditioning map, produced by the reference's own code:
`make_synthetic_map_factory` (terrain_diffusion/inference/synthetic_map.py:182-271, imported unmodified), its
`transform_perlin` (perlin_transform.py:42-45) and the WorldPipeline conditioning methods (world_pipeline.py:389-391,
821-903, extracted from the source with `ast` because the module builds the whole pipeline).

The factory imports pyfastnoiselite and rasterio.  The stand-in FastNoiseLite of tests/_minecraft_inputs.py is
installed as `pyfastnoiselite.pyfastnoiselite` (its values depend on the seed and every setting it is given, so matching
them pins the seed derivation and the coordinates), and `rasterio` is a stub that raises when called: the statistics
fixture of tests/_synthetic_inputs.py is written at the factory's cache path (`data/global/synthetic_map_stats.json`)
in a temporary working directory, so the statistics are never computed.  The golden therefore pins everything of the
map except the Perlin arithmetic itself, which the GPU tests pin to oracle/synthetic_map.py.

Stored (tests/golden/synthetic_golden.npz), per factory case: the map `f(i1, j1, i2, j2)` and `f.sample_raw(...)`
(fp64, as the reference returns it); per import case: `_conditioning_model_input` with the case's imports and without
them; `transform_perlin` of the knot noise per channel; `f.finalize` of the knot raw map; the numpy version.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_synthetic.py
"""
from __future__ import annotations

import ast
import os
import random
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])
sys.path[:0] = [str(ROOT), str(REF)]

from tests._minecraft_inputs import install_stand_in  # noqa: E402
from tests._synthetic_inputs import CASES, IMPORT_CASES, knot_noise, knot_raw, stats_fixture, write_stats  # noqa: E402

METHODS = ("_has_custom_conditioning_imports", "_sample_raw_conditioning", "_sample_custom_conditioning_channel",
           "_raw_conditioning_with_imports", "_conditioning_model_input")


def install_rasterio_stub() -> None:
    def _open(*a, **k):
        raise AssertionError("rasterio.open called: the statistics cache was not used")
    sys.modules["rasterio"] = types.SimpleNamespace(open=_open)


def conditioning_class():
    """A class holding the reference WorldPipeline's conditioning methods, nothing else."""
    src = (REF / "terrain_diffusion/inference/world_pipeline.py").read_text()
    cls = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "WorldPipeline")
    funcs = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in METHODS]
    assert len(funcs) == len(METHODS), "world_pipeline.py conditioning methods not found"
    body = ast.ClassDef(name="Conditioning", bases=[], keywords=[], body=funcs, decorator_list=[])
    mod = ast.fix_missing_locations(ast.Module(body=[body], type_ignores=[]))
    ns = {"np": np, "torch": torch}
    exec(compile(mod, "world_pipeline_extract", "exec", dont_inherit=True), ns)
    return ns["Conditioning"]


def make_factory(ref, case):
    seed, draw, fm, _ = CASES[case]
    random.seed(draw)
    return ref.make_synthetic_map_factory(frequency_mult=list(fm), seed=seed)


def main():
    install_stand_in()
    install_rasterio_stub()
    store = {"numpy_version": np.array(np.__version__)}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            os.makedirs("data/global")
            write_stats("data/global/synthetic_map_stats.json")
            from terrain_diffusion.inference import perlin_transform, synthetic_map as ref
            for name, (seed, draw, fm, win) in CASES.items():
                f = make_factory(ref, name)
                m = f(*win)
                assert isinstance(m, torch.Tensor) and m.dtype == torch.float32
                store[f"case.{name}.map"] = m.numpy()
                store[f"case.{name}.raw"] = np.asarray(f.sample_raw(*win))
                print(name, win, tuple(m.shape), store[f"case.{name}.raw"].dtype)
            Conditioning = conditioning_class()
            for name, (win, case, imports) in IMPORT_CASES.items():
                c = Conditioning()
                c.synthetic_map_factory = make_factory(ref, case)
                c.custom_conditioning_imports, c.custom_conditioning_import_origins = {}, {}
                c.custom_conditioning_default_values = {}
                store[f"import.{name}.plain"] = c._conditioning_model_input(*win).numpy()
                for ch, (values, origin, default) in imports.items():       # set_custom_conditioning_import's state
                    c.custom_conditioning_imports[ch] = np.asarray(values, np.float32).copy()
                    c.custom_conditioning_import_origins[ch] = origin
                    if default is not None:
                        c.custom_conditioning_default_values[ch] = float(default)
                store[f"import.{name}"] = c._conditioning_model_input(*win).numpy()
                print("import", name, win)
            stats = ref._load_stats_cache()
            noise = knot_noise()
            store["knots.raw"] = np.stack([perlin_transform.transform_perlin(
                noise[k], stats[f"noise_quantiles_{k}"], stats[f"base_image_quantiles_{k}"]) for k in range(5)])
            store["knots.finalize"] = np.asarray(make_factory(ref, "neg").finalize(knot_raw()))
        finally:
            os.chdir(cwd)
    assert stats_fixture()["n_quantiles"] == 64
    np.savez_compressed(HERE / "synthetic_golden.npz", **store)
    print("wrote", HERE / "synthetic_golden.npz", "numpy", np.__version__)


if __name__ == "__main__":
    main()
