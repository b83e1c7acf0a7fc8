"""CPU restatement of the explorer's detail view (explorer/server.py:188-270) in numpy, with the dtype of every
intermediate written out.  matplotlib is not needed; its four pieces the handlers use are restated here:

* `Normalize.__call__` (matplotlib >= 3.9, NumPy >= 2.1): the data stays fp32; vmin and vmax are NumPy float64 scalars,
  strong under NEP 50, so `resdat -= vmin` and `resdat /= (vmax - vmin)` each compute in fp64 and round once into the
  fp32 array; vmin == vmax fills every pixel, NaN included, with 0.
* `Colormap.__call__` on float input: x * 256 in x's dtype, 256 -> 255, below 0 -> the first entry, >= 256 -> the last,
  NaN -> the bad colour (0, 0, 0, 0), alpha 1 elsewhere; the fp64 table, rounded to fp32 by the handler's `.astype`.
* `ScalarMappable.to_rgba(bytes=True)` of an fp32 RGBA image (what `plt.imsave` passes to the PNG encoder): a pixel
  with any NaN channel becomes (0, 0, 0, 0) (matplotlib 3.8+), then uint8(trunc(fp32(x * 255))).
* `RdBu_r`: `terrain_diffusion_b200.inference.explorer.rdbu_r_lut` (`terrain`: `relief.terrain_lut`).

The relief is oracle/relief.py.  Pinned against the reference's own handlers by tests/golden/explorer_golden.npz; the
device kernels are checked against this module."""
from __future__ import annotations

import numpy as np

from oracle.relief import relief_map
from terrain_diffusion_b200.inference.explorer import CMAPS

LUT_SIZE = 256


def detail_window(ci: int, cj: int, detail_size: int, pan_i: int, pan_j: int) -> tuple[int, int, int, int]:
    """(i1, j1, i2, j2) the handlers pass to get() (server.py:199-203, 248-252)."""
    center_i, center_j = ci * 256 + pan_i, cj * 256 + pan_j
    half = detail_size // 2
    return center_i - half, center_j - half, center_i + half, center_j + half


def nan_range(plane: np.ndarray) -> tuple[float, float]:
    """server.py:207-209: Python floats of np.nanmin / np.nanmax (NaN for an all-NaN plane), vmax = vmin + 1 if equal."""
    finite = plane[~np.isnan(plane)]
    vmin, vmax = (float(finite.min()), float(finite.max())) if finite.size else (float("nan"), float("nan"))
    if vmax == vmin:
        vmax = vmin + 1
    return vmin, vmax


def normalize(plane: np.ndarray, vmin: float, vmax: float) -> np.ndarray:
    """fp32 [H, W]: Normalize(vmin, vmax)(plane)."""
    result = np.array(plane, dtype=np.float32, copy=True)
    v0, v1 = np.float64(vmin), np.float64(vmax)
    if v0 == v1:
        result.fill(0)
        return result
    with np.errstate(invalid="ignore", over="ignore"):
        result -= v0                                    # fp64 subtract, rounded into fp32
        result /= (v1 - v0)                             # fp64 divide, rounded into fp32
    return result


def colormap(x: np.ndarray, cmap: str) -> np.ndarray:
    """fp32 RGBA [..., 4]: plt.get_cmap(cmap)(x).astype(np.float32)."""
    lut = np.concatenate([CMAPS[cmap](), np.ones((LUT_SIZE, 1))], axis=1)
    xa = np.array(x, copy=True)
    with np.errstate(over="ignore", invalid="ignore"):
        xa *= LUT_SIZE
    xa[xa == LUT_SIZE] = LUT_SIZE - 1
    bad = np.isnan(xa)
    idx = np.where(bad | (xa < 0), 0, np.where(xa >= LUT_SIZE, LUT_SIZE - 1, np.nan_to_num(xa))).astype(np.int64)
    rgba = lut[idx]
    rgba[bad] = 0.0
    return rgba.astype(np.float32)


def to_rgba_bytes(rgba: np.ndarray) -> np.ndarray:
    """uint8 [H, W, 4]: ScalarMappable.to_rgba(rgba, bytes=True) of an fp32 RGBA image in [0, 1] (or NaN)."""
    xx = np.array(rgba, dtype=np.float32, copy=True)
    xx[np.isnan(xx).any(axis=2), :] = 0
    return (xx * 255).astype(np.uint8)


def png_rgba(rgba: np.ndarray) -> np.ndarray:
    """uint8 [H, W, 4] that `_png_response(rgba)` (server.py:67-71) encodes: np.clip(rgba, 0, 1), then imsave's
    to_rgba(bytes=True)."""
    return to_rgba_bytes(np.clip(rgba, 0, 1))


def colour_plane(plane: np.ndarray, cmap: str) -> np.ndarray:
    """uint8 [H, W, 4]: the elevation / temperature branch (server.py:206-218) of an fp32 plane."""
    plane = np.asarray(plane, dtype=np.float32)
    vmin, vmax = nan_range(plane)
    return png_rgba(colormap(normalize(plane, vmin, vmax), cmap))


def relief_rgba(relief_rgb: np.ndarray) -> np.ndarray:
    """uint8 [H, W, 4]: the relief branch (server.py:223-228) of get_relief_map's fp32 RGB."""
    rgba = np.concatenate([np.clip(relief_rgb, 0, 1), np.ones((*relief_rgb.shape[:2], 1), dtype=np.float32)], axis=-1)
    return png_rgba(rgba)


def detail_image(elev: np.ndarray, temp: np.ndarray | None, mode: str, native_resolution: float) -> np.ndarray:
    """uint8 [H, W, 4]: `detail_png`'s picture of one window by mode (server.py:206-228)."""
    if mode == "elevation":
        return colour_plane(elev, "terrain")
    if mode == "temperature" and temp is not None:
        return colour_plane(temp, "RdBu_r")
    with np.errstate(invalid="ignore"):
        return relief_rgba(relief_map(elev, resolution=native_resolution))


def detail_raw_body(elev: np.ndarray, temp: np.ndarray | None) -> bytes:
    """`detail_raw`'s body (server.py:253-260): int16-LE elevation (floor, clip), then fp32-LE temperature."""
    with np.errstate(invalid="ignore"):
        e16 = np.clip(np.floor(np.asarray(elev, dtype=np.float32)), -32768, 32767).astype("<i2")
    return e16.tobytes() + (b"" if temp is None else np.asarray(temp).astype("<f4").tobytes())
