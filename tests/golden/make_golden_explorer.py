"""Golden vectors for the explorer's detail view, produced by the reference's own handlers `detail_png`, `detail_raw`
and `_png_response` (terrain_diffusion/inference/explorer/server.py).  The server imports flask and matplotlib, which are
absent here, so the three functions are extracted from its source with `ast` (their route decorators dropped) and run
with stand-ins:

* `request.args`: Flask's `args.get(key, default, type)` over the case's arguments;
* `_get_pipeline()`: a world whose `get()` returns the seeded analytic planes of tests/_explorer_inputs.py on absolute
  coordinates (or, for the plane cases, one given plane) as CPU tensors, and records the window it was asked for;
* `Response` and `jsonify` (which raises, so a handler error cannot pass for a result);
* `plt.get_cmap` returning `Colormap`, a restatement of matplotlib 3.9's `Colormap._get_rgba_and_mask` over the
  restated `terrain` / `RdBu_r` tables; `matplotlib.colors.Normalize`, restated from matplotlib 3.9's
  `Normalize.__call__` / `process_value`;
* `plt.imsave`, which records the uint8 RGBA that `ScalarMappable.to_rgba(arr, bytes=True)` hands to PIL (restated:
  a pixel with a NaN channel becomes 0 in all four channels, then `(x * 255).astype(np.uint8)`);
* `get_relief_map`: the reference's own, extracted as tests/golden/make_golden_relief.py does, recording its fp32 RGB.

These stand-ins are written separately from oracle/explorer.py, which tests/test_explorer_cpu.py holds to this file.
Stored (tests/golden/explorer_golden.npz): per case the window get() was asked for, the image (uint8 RGBA, not PNG
bytes) and for the relief the fp32 RGB, or the raw body and its headers; the numpy version.

    TERRAIN_DIFFUSION_REF=<checkout of the original project> python tests/golden/make_golden_explorer.py
"""
from __future__ import annotations

import __future__
import ast
import io
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])
sys.path[:0] = [str(ROOT)]

from terrain_diffusion_b200.inference.explorer import rdbu_r_lut  # noqa: E402
from terrain_diffusion_b200.inference.relief import terrain_lut  # noqa: E402
from tests._explorer_inputs import HANDLER_CASES, NATIVE_RESOLUTION, PLANE_CASES, plane_case, world_planes  # noqa: E402
from tests.golden.make_golden_relief import reference_get_relief_map  # noqa: E402


class Normalize:
    """matplotlib 3.9 colors.Normalize, the parts `Normalize(vmin=, vmax=)(x)` runs."""

    def __init__(self, vmin=None, vmax=None, clip=False):
        self.vmin, self.vmax, self.clip = self._sanitize(vmin), self._sanitize(vmax), clip

    @staticmethod
    def _sanitize(value):
        try:
            return value.item()
        except AttributeError:
            return float(value)

    @staticmethod
    def process_value(value):
        is_scalar = not np.iterable(value)
        if is_scalar:
            value = [value]
        dtype = np.min_scalar_type(value)
        if np.issubdtype(dtype, np.integer) or dtype.type is np.bool_:
            dtype = np.promote_types(dtype, np.float32)
        mask = np.ma.getmask(value)
        data = np.asarray(value)
        return np.ma.array(data, mask=mask, dtype=dtype, copy=True), is_scalar

    def __call__(self, value):
        result, _ = self.process_value(value)
        (vmin,), _ = self.process_value(self.vmin)
        (vmax,), _ = self.process_value(self.vmax)
        if vmin == vmax:
            result.fill(0)
        elif vmin > vmax:
            raise ValueError("minvalue must be less than or equal to maxvalue")
        else:
            resdat = result.data
            resdat -= vmin
            resdat /= (vmax - vmin)
            result = np.ma.array(resdat, mask=result.mask, copy=False)
        return result


class Colormap:
    """matplotlib 3.9 Colormap.__call__ (alpha None, bytes False) over an N x 3 fp64 table: lut rows N, N+1, N+2 are
    under (= first entry), over (= last entry) and bad ((0, 0, 0, 0))."""

    def __init__(self, table):
        self.N = len(table)
        self._lut = np.ones((self.N + 3, 4), float)
        self._lut[:-3, :3] = table
        self._lut[self.N] = self._lut[0]
        self._lut[self.N + 1] = self._lut[self.N - 1]
        self._lut[self.N + 2] = 0.0
        self._i_under, self._i_over, self._i_bad = self.N, self.N + 1, self.N + 2

    def __call__(self, X):
        xa = np.array(X, copy=True)
        if xa.dtype.kind == "f":
            xa *= self.N
            xa[xa == self.N] = self.N - 1
        mask_under = xa < 0
        mask_over = xa >= self.N
        mask_bad = X.mask if np.ma.is_masked(X) else np.isnan(xa)
        with np.errstate(invalid="ignore"):
            xa = xa.astype(int)
        xa[mask_under] = self._i_under
        xa[mask_over] = self._i_over
        xa[mask_bad] = self._i_bad
        return self._lut.take(xa, axis=0, mode="clip")


def to_rgba_bytes(x):
    """ScalarMappable.to_rgba(x, bytes=True) for an (M, N, 4) float image (matplotlib 3.8+)."""
    xx = x
    if xx.dtype.kind == "f":
        if np.any(nans := np.isnan(x)):
            xx = xx.copy()
            xx[np.any(nans, axis=2), :] = 0
        if xx.max() > 1 or xx.min() < 0:
            raise ValueError("Floating point image RGB values must be in the 0..1 range.")
        xx = (xx * 255).astype(np.uint8)
    return xx


class Response:
    def __init__(self, data, mimetype=None):
        self.data, self.mimetype, self.headers = data, mimetype, {}


def jsonify(payload):
    raise RuntimeError(f"the handler failed: {payload}")


class Args(dict):
    def get(self, key, default=None, type=None):
        if key not in self:
            return default
        return type(str(self[key])) if type is not None else self[key]


class FakeWorld:
    native_resolution = NATIVE_RESOLUTION

    def __init__(self, planes):
        self.planes, self.windows = planes, []

    def get(self, i1, j1, i2, j2):
        self.windows.append((i1, j1, i2, j2))
        elev, climate = self.planes(i1, j1, i2, j2)
        return {"elev": torch.from_numpy(elev), "climate": torch.from_numpy(climate)}


def reference_handlers():
    src = (REF / "terrain_diffusion/inference/explorer/server.py").read_text()
    body = [n for n in ast.parse(src).body
            if isinstance(n, ast.FunctionDef) and n.name in ("_png_response", "detail_png", "detail_raw")]
    assert len(body) == 3, "_png_response / detail_png / detail_raw not found"
    for n in body:
        n.decorator_list = []
    code = compile(ast.Module(body=body, type_ignores=[]), "server_extract", "exec",
                   flags=__future__.annotations.compiler_flag, dont_inherit=True)
    state = SimpleNamespace(world=None, args=None, images=[], relief=[])
    ref_relief = reference_get_relief_map()

    def get_relief_map(*a, **k):
        out = ref_relief(*a, **k)
        state.relief.append(out)
        return out

    def imsave(fname, arr, format=None):
        state.images.append(to_rgba_bytes(arr))
        fname.write(b"PNG stand-in")

    cmaps = {"terrain": Colormap(terrain_lut()), "RdBu_r": Colormap(rdbu_r_lut())}
    ns = {"io": io, "np": np, "Response": Response, "jsonify": jsonify, "get_relief_map": get_relief_map,
          "matplotlib": SimpleNamespace(colors=SimpleNamespace(Normalize=Normalize)),
          "plt": SimpleNamespace(get_cmap=cmaps.__getitem__, imsave=imsave),
          "request": SimpleNamespace(args=None), "_get_pipeline": lambda: state.world}
    exec(code, ns)

    def run(name, world, args):
        state.world, state.images, state.relief = world, [], []
        ns["request"].args = Args(args)
        resp = ns[name]()
        assert isinstance(resp, Response), resp
        return resp, state

    return run


def main():
    run = reference_handlers()
    out = {"numpy_version": np.array(np.__version__)}
    for name, (kind, endpoint, args) in HANDLER_CASES.items():
        world = FakeWorld(lambda i1, j1, i2, j2, kind=kind: world_planes(kind, i1, j1, i2, j2))
        resp, state = run("detail_png" if endpoint == "png" else "detail_raw", world, args)
        assert len(world.windows) == 1
        out[f"{name}.window"] = np.array(world.windows[0], np.int64)
        if endpoint == "png":
            assert resp.mimetype == "image/png" and len(state.images) == 1
            out[f"{name}.image"] = state.images[0]
            if state.relief:
                out[f"{name}.relief_rgb"] = state.relief[0]
            print(name, world.windows[0], state.images[0].shape, "transparent px",
                  int((state.images[0][..., 3] == 0).sum()))
        else:
            h = resp.headers
            assert h["Access-Control-Expose-Headers"] == "X-Height, X-Width, X-Has-Temp"
            out[f"{name}.body"] = np.frombuffer(resp.data, np.uint8).copy()
            out[f"{name}.headers"] = np.array([int(h["X-Height"]), int(h["X-Width"]), int(h["X-Has-Temp"])], np.int64)
            print(name, world.windows[0], "body bytes", len(resp.data), "headers", out[f"{name}.headers"])
    for name in PLANE_CASES:
        plane, cmap = plane_case(name)
        zeros = np.zeros_like(plane)
        if cmap == "terrain":
            planes = lambda *_: (plane, np.stack([zeros] * 5))
        else:
            planes = lambda *_: (zeros, np.stack([plane] + [zeros] * 4))
        mode = "elevation" if cmap == "terrain" else "temperature"
        with np.errstate(invalid="ignore", over="ignore"):
            _, state = run("detail_png", FakeWorld(planes), {"mode": mode})
        out[f"plane.{name}.image"] = state.images[0]
        print("plane", name, plane.shape, cmap, "distinct colours", len(np.unique(state.images[0].reshape(-1, 4), axis=0)))
    np.savez_compressed(HERE / "explorer_golden.npz", **out)
    print("wrote", HERE / "explorer_golden.npz", "numpy", np.__version__)


if __name__ == "__main__":
    main()
