"""CPU restatement of the shaded relief map (get_relief_map, inference/relief_map.py:64-199) in numpy + scipy, with the
dtype of every intermediate written out: fp32 arrays, Python-float scalars that take the array's dtype (NEP 50), the
float64 `np.deg2rad` scalars that promote the hillshade mix to fp64.  The `terrain` colormap is the restated table of
terrain_diffusion_b200.inference.relief (matplotlib is not needed).  Pinned against the reference's own function by
tests/golden/relief_golden.npz; the device kernels are checked against this module."""
from __future__ import annotations

import numpy as np
from scipy.ndimage import gaussian_filter

from terrain_diffusion_b200.inference.relief import LUT_SIZE, terrain_lut

_LUT = None


def terrain_cmap(x) -> np.ndarray:
    """matplotlib Colormap.__call__ on float input: RGBA fp64.  x*N (in x's dtype), x == N -> N-1, below 0 -> the
    first entry, >= N -> the last, NaN -> the bad colour (0, 0, 0, 0)."""
    global _LUT
    if _LUT is None:
        _LUT = np.concatenate([terrain_lut(), np.ones((LUT_SIZE, 1))], axis=1)
    xa = np.array(x, copy=True)
    xa *= LUT_SIZE
    xa[xa == LUT_SIZE] = LUT_SIZE - 1
    bad = np.isnan(xa)
    idx = np.where(bad | (xa < 0), 0, np.where(xa >= LUT_SIZE, LUT_SIZE - 1, np.nan_to_num(xa))).astype(np.int64)
    rgba = _LUT[idx]
    rgba[bad] = 0.0
    return rgba


def _hillshade(z: np.ndarray, grad_div: float, az_deg: float, alt_deg: float) -> np.ndarray:
    gy, gx = np.gradient(z)                                   # fp32, edge order 1
    gy, gx = gy / grad_div, gx / grad_div                     # Python float -> fp32 division
    slope = np.float32(np.pi / 2.0) - np.arctan(np.hypot(gx, gy))
    aspect = np.arctan2(gy, -gx)
    az, alt = np.deg2rad(az_deg), np.deg2rad(alt_deg)         # float64 scalars
    mix = np.sin(alt) * np.sin(slope).astype(np.float64) \
        + np.cos(alt) * np.cos(slope).astype(np.float64) * np.cos(az - aspect.astype(np.float64))
    return np.clip(mix, 0.0, 1.0).astype(np.float32)


def colour_range(elev: np.ndarray, vmin=None, vmax=None) -> tuple[float, float]:
    """(_vmin, _vmax) of relief_map.py:135-142: the nan-range of max(0, elev) unless both bounds are given."""
    if vmin is not None and vmax is not None:
        return max(0.0, float(vmin)), float(vmax)
    land = np.maximum(np.float32(0), elev)
    finite = land[~np.isnan(land)]
    lo, hi = (float(finite.min()), float(finite.max())) if finite.size else (float("nan"), float("nan"))
    if not (np.isfinite(lo) and np.isfinite(hi)) or lo == hi:
        return 0.0, 1.0
    return lo, hi


def relief_parts(elevation, *, azimuths=(315.0, 45.0, 135.0, 225.0), sigma_large=6.0, sigma_small=1.2,
                 resolution=90, relief=1.0, vmin=None, vmax=None):
    """{'rgb': fp32 [H, W, 3], 'arg': the fp32 colormap argument [H, W], 'gain': the fp32 intensity factor [H, W],
    'ocean': bool [H, W]} for elevation, with climate / biome / flow / rgb all None."""
    elev = np.asarray(elevation, dtype=np.float32)
    az_deg = float(azimuths[0]) if isinstance(azimuths, (tuple, list)) and len(azimuths) > 0 else 315.0
    nan = np.isnan(elev)
    filled = elev
    if nan.any():
        finite = np.sort(elev[~nan])
        if finite.size == 0:
            fill = 0.0
        elif finite.size % 2:
            fill = float(finite[finite.size // 2])
        else:
            fill = float((finite[finite.size // 2 - 1] + finite[finite.size // 2]) / np.float32(2))
        filled = np.where(nan, np.float32(fill if np.isfinite(fill) else 0.0), elev)
    grad_div = 15 * resolution / 90
    hs = [_hillshade(gaussian_filter(filled, sigma=s), grad_div, az_deg, 45.0) for s in (sigma_large, sigma_small)]
    hill = np.clip(np.float32(0.75) * hs[0] + np.float32(0.25) * hs[1], np.float32(0), np.float32(1))
    hill = np.power(hill, np.float32(0.85))

    lo, hi = colour_range(elev, vmin, vmax)
    land = np.maximum(np.float32(0), elev)
    norm = (land - np.float32(lo)) / np.float32(hi - lo + 1e-8)
    with np.errstate(invalid="ignore"):
        arg = np.clip(np.power(norm, np.float32(0.7)), np.float32(0), np.float32(1))
    if lo == 0.0:
        arg = np.float32(0.25) + arg * np.float32(0.75)
    base = terrain_cmap(arg)[..., :3].astype(np.float32)

    gain = np.float32(relief) * (np.float32(0.35) + np.float32(0.65) * hill) + np.float32(1 - relief)
    rgb = np.clip(base * gain[..., None], np.float32(0), np.float32(1))
    rgb[nan] = np.nan
    ocean = filled < 0
    t = np.power(np.clip(-filled / np.float32(10000.0), np.float32(0), np.float32(1)), np.float32(0.7))
    coast = np.array([0.68, 0.88, 1.00], dtype=np.float32)
    deep = np.array([0.00, 0.10, 0.45], dtype=np.float32)
    sea = (np.float32(1) - t)[..., None] * coast + t[..., None] * deep
    rgb = np.where(ocean[..., None], sea, rgb).astype(np.float32)
    return {"rgb": rgb, "arg": arg, "gain": gain, "ocean": ocean}


def relief_map(elevation, **kw) -> np.ndarray:
    return relief_parts(elevation, **kw)["rgb"]
