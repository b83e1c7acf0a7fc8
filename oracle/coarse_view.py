"""CPU restatement of the explorer's coarse map (explorer/server.py:58-185) and the random sampler's land search
(random_sampler.py:61-119) in numpy, with the dtype of every intermediate written out.  matplotlib is not needed: the
pieces the handlers use are oracle/explorer.py's (`Normalize`, `to_rgba(bytes=True)`); `Colormap` takes its table as an
argument here, because viridis is not restated.

* `_coarse_channel` / `normalize_tensor`: torch CPU fp32, x = v / (w + fp32(1e-8)) or v / w, then for channels 0 and 1
  np.sign(x) * np.square(x) in fp32 (torch.sign * torch.square gives the same bits: +0 for +-0, NaN for NaN).
* The display plane of channel 4: np.log1p(np.maximum(x, 0)) in fp32.
* The filters: an fp32 array compared with a Python float, which NumPy 2 rounds to fp32 (NEP 50); `rgba[~mask, :3] *=
  0.3` multiplies in fp32.
* np.round(x, 2) of fp32: x * 100 in fp32, rint, / 100 in fp32.
* The land fraction: torch's CPU fp32 mean of 0 / 1 values, sum / numel correctly rounded, compared in fp64.

Pinned against the reference's own handlers by tests/golden/coarse_view_golden.npz; the device kernels are checked
against this module."""
from __future__ import annotations

import numpy as np

from oracle.explorer import nan_range, normalize, png_rgba

CHANNEL_NAMES = ["Elev", "p5", "Temp", "T std", "Precip", "Precip CV"]
FILTERABLE = (0, 2, 3, 4, 5)
LUT_SIZE = 256


def signed_square(x: np.ndarray) -> np.ndarray:
    return (np.sign(x) * np.square(x)).astype(np.float32)


def coarse_planes(sums: np.ndarray, eps: bool = True) -> np.ndarray:
    """fp32 [6, h, w]: the real-unit channels of a [7, h, w] (sum v*w, sum w) slice."""
    sums = np.asarray(sums, dtype=np.float32)
    w = sums[6:7] + np.float32(1e-8) if eps else sums[6:7]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        x = (sums[:6] / w).astype(np.float32)
        x[:2] = signed_square(x[:2])
    return x


def display(planes: np.ndarray, channel: int) -> np.ndarray:
    """fp32 [h, w]: what the image shows (server.py:113)."""
    data = planes[channel]
    if channel != 4:
        return data
    with np.errstate(invalid="ignore"):
        return np.log1p(np.maximum(data, np.float32(0))).astype(np.float32)


def colormap(x: np.ndarray, table: np.ndarray) -> np.ndarray:
    """fp32 RGBA [..., 4]: Colormap over the fp64 [256, 3] `table` (alpha 1), `.astype(np.float32)`."""
    lut = np.concatenate([np.asarray(table, np.float64), np.ones((LUT_SIZE, 1))], axis=1)
    xa = np.array(x, copy=True)
    with np.errstate(over="ignore", invalid="ignore"):
        xa *= LUT_SIZE
    xa[xa == LUT_SIZE] = LUT_SIZE - 1
    bad = np.isnan(xa)
    idx = np.where(bad | (xa < 0), 0, np.where(xa >= LUT_SIZE, LUT_SIZE - 1, np.nan_to_num(xa))).astype(np.int64)
    rgba = lut[idx]
    rgba[bad] = 0.0
    return rgba.astype(np.float32)


def filter_mask(planes: np.ndarray, filters: dict | None) -> np.ndarray | None:
    """bool [h, w] of the cells that pass every given bound (server.py:122-136), or None without an active filter."""
    filters = {ch: b for ch, b in (filters or {}).items() if ch in FILTERABLE}
    if not any(v is not None for b in filters.values() for v in b):
        return None
    mask = np.ones(planes.shape[1:], dtype=bool)
    with np.errstate(invalid="ignore", over="ignore"):
        for ch, (lo, hi) in filters.items():
            if lo is not None:
                mask &= planes[ch] >= lo
            if hi is not None:
                mask &= planes[ch] <= hi
    return mask


def coarse_image(planes: np.ndarray, channel: int, table: np.ndarray, filters: dict | None = None,
                 shown: np.ndarray | None = None) -> tuple[np.ndarray, float, float]:
    """(uint8 RGBA [h, w, 4], vmin, vmax) of `coarse_png` (server.py:112-139) on the eps planes; `shown` replaces the
    display plane (the device's log1p plane, to compare the rest of the chain bit for bit)."""
    shown = display(planes, channel) if shown is None else np.asarray(shown, np.float32)
    vmin, vmax = nan_range(shown)
    rgba = colormap(normalize(shown, vmin, vmax), table)
    mask = filter_mask(planes, filters)
    if mask is not None:
        rgba[~mask, :3] *= 0.3
    return png_rgba(rgba), vmin, vmax


def coarse_data(planes: np.ndarray) -> np.ndarray:
    """fp32 [6, h, w]: np.round(x, 2) of every channel (server.py:159)."""
    return np.round(np.asarray(planes, np.float32), 2)


def coarse_stats(planes: np.ndarray) -> dict:
    """`coarse_stats`'s dict (server.py:175-183)."""
    out = {}
    for ch, name in enumerate(CHANNEL_NAMES):
        fin = planes[ch][~np.isnan(planes[ch])]
        lo, hi = (float(fin.min()), float(fin.max())) if fin.size else (float("nan"), float("nan"))
        out[ch] = {"name": name, "min": round(lo, 3), "max": round(hi, 3)}
    return out


def land_tiles(sums: np.ndarray, ci0: int, cj0: int, detail_size: int, min_land_frac: float) -> list:
    """`valid_tiles` of sample_land_tiles (random_sampler.py:75-93) for a [7, H, W] slice whose cell (0, 0) is
    (ci0, cj0): window counts from a summed-area table, fp32(count / n) >= min_land_frac in fp64."""
    land = (coarse_planes(sums, eps=False)[0] > 0).astype(np.int64)
    H, W = land.shape
    half = (detail_size // 256) // 2
    n = (2 * half) ** 2
    if H - 2 * half <= 0 or W - 2 * half <= 0 or n == 0:
        return []
    sat = np.zeros((H + 1, W + 1), np.int64)
    sat[1:, 1:] = land.cumsum(0).cumsum(1)
    k = 2 * half
    count = sat[k:, k:] - sat[:-k, k:] - sat[k:, :-k] + sat[:-k, :-k]          # [H - k + 1, W - k + 1]
    count = count[:H - k, :W - k]                                             # windows starting at io < H - 2 half
    frac = count.astype(np.float32) / np.float32(n)
    io, jo = np.nonzero(frac.astype(np.float64) >= float(min_land_frac))
    return [(ci0 + half + int(i), cj0 + half + int(j)) for i, j in zip(io, jo)]


def climate_info(sums_cell: np.ndarray) -> dict:
    """get_coarse_climate_info's dict (random_sampler.py:102-119) of a [7, 1, 1] slice."""
    p = coarse_planes(sums_cell, eps=False)
    return {"temp": float(p[2, 0, 0]), "temp_std": float(p[3, 0, 0]), "precip": float(p[4, 0, 0]),
            "precip_cv": float(p[5, 0, 0])}
