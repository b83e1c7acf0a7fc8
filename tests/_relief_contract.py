"""What csrc/tdx_relief.cu's shade kernel promises, restated operation by operation in numpy, and the tolerance rule of
the shaded relief map against oracle/relief.py.

oracle/relief.py is the reference's numpy program: fp32 ufuncs whose transcendentals (numpy's SIMD arctan, sin, cos,
power) are not correctly rounded, so the device can only be held to it within a bound.  `shade` below is instead the
kernel's own arithmetic: the same fp32 and fp64 operations in the same order, each rounded once, with every
transcendental evaluated in fp64 and rounded to fp32 (or, for the cosine inside the hillshade mix, kept in fp64).
numpy's fp32 / fp64 add, multiply, divide and sqrt are correctly rounded like the kernel's `__f*_rn` / `__d*_rn`, so
everything except the fp64 transcendentals is reproduced bit for bit.

Neither CUDA's fp64 transcendentals nor the host's are correctly rounded (a few ulps each), so a pixel is excused where
a value rounded from fp64 to fp32 lies within ULPS fp64 ulps of an fp32 rounding midpoint (there the two libraries may
round to different fp32 neighbours), or where the fp64 hillshade mix lies within that margin of its clip at 0 or 1.  The
colormap index, the fp32 clips and the `filled < 0` test act on fp32 values that are already pinned bit for bit by the
rule above (`filled` is an input value, never computed), so they need no margin of their own.  Every other pixel must
match bit for bit; excused pixels are still held to `compare` against the oracle.
"""
from __future__ import annotations

import numpy as np
from scipy.ndimage import gaussian_filter

from terrain_diffusion_b200.inference.relief import ALTITUDE_DEG, LUT_SIZE, terrain_lut

F32, F64 = np.float32, np.float64
ULPS = 8                         # fp64 ulps between CUDA's and the host's transcendentals, both sides together
MIX_MARGIN = ULPS * 2.0 ** -53   # the hillshade mix: terms of magnitude <= 1, an error of ULPS half-ulps of 1
TOL, BOUNDARY = 2e-5, 1e-4       # the rule against the oracle (see `compare`)
COAST = np.array([0.68, 0.88, 1.00], dtype=F32)
DEEP = np.array([0.00, 0.10, 0.45], dtype=F32)
LUT32 = terrain_lut().astype(F32)


def near_f32_midpoint(v, margin) -> np.ndarray:
    """fp64 `v` lies within `margin` of a point halfway between two adjacent fp32 values (non-finite v: never)."""
    v = np.asarray(v, dtype=F64)
    with np.errstate(over="ignore", invalid="ignore"):
        f = v.astype(F32)
        lo = np.nextafter(f, F32(-np.inf)).astype(F64)
        hi = np.nextafter(f, F32(np.inf)).astype(F64)
        f = f.astype(F64)
        d = np.minimum(np.abs(v - (f + lo) / 2), np.abs(v - (f + hi) / 2))   # both sums exact in fp64
    return np.isfinite(v) & np.isfinite(f) & (d <= margin)


def _ulps(v):
    return ULPS * np.spacing(np.abs(np.asarray(v, dtype=F64)))


def _rounded(v64, excused):
    """fp32 of an fp64 transcendental result; marks `excused` where another library's result may round differently."""
    excused |= near_f32_midpoint(v64, _ulps(v64))
    return v64.astype(F32)


def pow_f32(x, e, excused):
    """The kernel's pow_f32: fp32(pow(fp64(x), fp64(e)))."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return _rounded(np.power(np.asarray(x, F32).astype(F64), F64(F32(e))), excused)


def clip01(v):
    """v < 0 -> 0, v > 1 -> 1, NaN stays NaN (the kernel's clip01, numpy's np.clip)."""
    return np.where(v < 0, v.dtype.type(0), np.where(v > 1, v.dtype.type(1), v))


def gradient(p):
    """np.gradient of an fp32 plane, edge order 1, written out: (dy, dx)."""
    dy, dx = np.empty_like(p), np.empty_like(p)
    with np.errstate(invalid="ignore", over="ignore"):
        dy[0], dy[-1] = p[1] - p[0], p[-1] - p[-2]
        dy[1:-1] = (p[2:] - p[:-2]) * F32(0.5)
        dx[:, 0], dx[:, -1] = p[:, 1] - p[:, 0], p[:, -1] - p[:, -2]
        dx[:, 1:-1] = (p[:, 2:] - p[:, :-2]) * F32(0.5)
    return dy, dx


def hillshade(p, grad_div, az, sin_alt, cos_alt, why):
    """The kernel's hillshade() over a whole fp32 plane; ORs its excuses into why['rounding'] and why['clip']."""
    dy, dx = gradient(p)
    with np.errstate(invalid="ignore", over="ignore"):
        dy, dx = dy / F32(grad_div), dx / F32(grad_div)
        ddx, ddy = dx.astype(F64), dy.astype(F64)
        hyp = np.sqrt(ddx * ddx + ddy * ddy).astype(F32)
        slope = F32(np.pi / 2) - _rounded(np.arctan(hyp.astype(F64)), why["rounding"])
        aspect = _rounded(np.arctan2(ddy, -ddx), why["rounding"])
        sin_s = _rounded(np.sin(slope.astype(F64)), why["rounding"]).astype(F64)
        cos_s = _rounded(np.cos(slope.astype(F64)), why["rounding"]).astype(F64)
        hs = F64(sin_alt) * sin_s + (F64(cos_alt) * cos_s) * np.cos(F64(az) - aspect.astype(F64))
    inside = (hs >= 0) & (hs <= 1)
    why["rounding"] |= inside & near_f32_midpoint(hs, MIX_MARGIN)
    why["clip"] |= (np.abs(hs) <= MIX_MARGIN) | (np.abs(hs - 1) <= MIX_MARGIN)
    return clip01(hs).astype(F32)


def decode_range(stats, user_range, vmin, denom, vmin_is_zero):
    """(vmin fp32, denom fp32, vmin is zero) as the shade kernel forms them: from tdx_relief_stats' buffer unless
    user_range, with the fallback range (0, 1) when an extremum is not finite or they are equal."""
    if user_range:
        return F32(vmin), F32(denom), bool(vmin_is_zero)
    lo, hi = decode_stats(stats)
    if is_fallback(lo, hi):
        dlo, dhi = 0.0, 1.0
    else:
        dlo, dhi = float(lo), float(hi)
    return F32(dlo), F32(dhi - dlo + 1e-8), dlo == 0.0


def decode_stats(stats):
    """(nanmin, nanmax) fp32 of max(0, x) from tdx_relief_stats' uint32 buffer: ~stats[1] and stats[2] as float bits."""
    s = np.asarray(stats).astype(np.int64) & 0xFFFFFFFF
    return (np.array([~s[1] & 0xFFFFFFFF], np.uint32).view(F32)[0], np.array([s[2]], np.uint32).view(F32)[0])


def is_fallback(lo, hi) -> bool:
    return not (np.isfinite(lo) and np.isfinite(hi)) or hi == lo


def shade(elev, blurred, stats, *, replace_nan, nan_fill, grad_div, az, sin_alt, cos_alt, relief, one_minus_relief,
          user_range, vmin, denom, vmin_is_zero):
    """tdx_relief_shade with these arguments (scalars as the C ABI receives them: float -> fp32, double -> fp64).
    Returns {'rgb': fp32 [H, W, 3], 'xa': the fp32 colormap argument x 256, 'gain': the fp32 intensity factor,
    'ocean': bool, 'excused': bool [H, W], 'why': {reason: bool [H, W]} before narrowing to the pixels it decides}."""
    elev = np.asarray(elev, F32)
    h, w = elev.shape
    why = {k: np.zeros((h, w), bool) for k in ("rounding", "clip", "colour power", "ocean power")}
    raw_nan = np.isnan(elev)
    filled = np.where(raw_nan & bool(replace_nan), F32(nan_fill), elev)
    hs_l = hillshade(blurred[0], grad_div, az, sin_alt, cos_alt, why)
    hs_s = hillshade(blurred[1], grad_div, az, sin_alt, cos_alt, why)
    hill = pow_f32(clip01(F32(0.75) * hs_l + F32(0.25) * hs_s), 0.85, why["rounding"])

    lo, dn, zero = decode_range(stats, user_range, vmin, denom, vmin_is_zero)
    land = np.where(raw_nan, elev, np.where(elev > 0, elev, F32(0)))
    with np.errstate(invalid="ignore", over="ignore"):
        norm = (land - lo) / dn
    c = clip01(pow_f32(norm, 0.7, why["colour power"]))
    if zero:
        c = F32(0.25) + c * F32(0.75)
    xa = c * F32(LUT_SIZE)
    idx = np.where(np.isnan(xa) | (xa < 0), 0, np.where(xa >= LUT_SIZE, LUT_SIZE - 1, np.nan_to_num(xa)))
    base = np.where(np.isnan(xa)[..., None], F32(0), LUT32[idx.astype(np.int64)])

    gain = F32(relief) * (F32(0.35) + F32(0.65) * hill) + F32(one_minus_relief)
    with np.errstate(invalid="ignore"):
        rgb = np.where(raw_nan[..., None], F32(np.nan), clip01(base * gain[..., None]))
    ocean = filled < 0
    with np.errstate(invalid="ignore", over="ignore"):
        t = pow_f32(clip01(-filled / F32(10000.0)), 0.7, why["ocean power"])
    sea = (F32(1) - t)[..., None] * COAST + t[..., None] * DEEP
    rgb = np.where(ocean[..., None], sea, rgb).astype(F32)
    land_px = ~ocean & ~raw_nan
    excused = (land_px & (why["rounding"] | why["clip"] | why["colour power"])) | (ocean & why["ocean power"])
    return {"rgb": rgb, "xa": xa, "gain": gain, "ocean": ocean, "excused": excused, "why": why}


def encode_stats(elev):
    """The uint32 [3] buffer tdx_relief_stats promises for `elev`: NaN count, ~bits(nanmin), bits(nanmax) of max(0, x)
    with -0 and negatives as +0; with no non-NaN value the minimum is +inf and the maximum +0."""
    x = np.asarray(elev, F32).reshape(-1)
    fin = x[~np.isnan(x)]
    land = np.where(fin > 0, fin, F32(0))
    lo = land.min() if land.size else F32(np.inf)
    hi = land.max() if land.size else F32(0)
    lo_bits = int(np.array([lo], F32).view(np.uint32)[0])
    hi_bits = int(np.array([hi], F32).view(np.uint32)[0])
    return np.array([int(np.isnan(x).sum()), ~lo_bits & 0xFFFFFFFF, hi_bits], np.uint32)


def nan_fill(elev) -> float:
    """The reference's NaN replacement: np.nanmedian of the fp32 values (even count: the fp32 mean of the middle two),
    0.0 when it is not finite or there is no value."""
    fin = np.sort(elev[~np.isnan(elev)])
    n = fin.size
    if n == 0:
        return 0.0
    m = float(fin[n // 2]) if n % 2 else float((fin[n // 2 - 1] + fin[n // 2]) / F32(2))
    return m if np.isfinite(m) else 0.0


def shade_args(elev, *, azimuths=(315.0, 45.0, 135.0, 225.0), sigma_large=6.0, sigma_small=1.2, resolution=90,
               relief=1.0, vmin=None, vmax=None):
    """The arguments get_relief_map passes tdx_relief_shade for `elev` (inference/relief.py `_relief`), with the
    blurred planes from scipy (which tdx_relief_gaussian matches bit for bit) and the statistics `encode_stats` gives."""
    elev = np.asarray(elev, F32)
    nan = np.isnan(elev)
    has_nan = bool(nan.any())
    fill = nan_fill(elev) if has_nan else 0.0
    filled = np.where(nan, F32(fill), elev) if has_nan else elev
    with np.errstate(invalid="ignore", over="ignore"):
        blurred = np.stack([gaussian_filter(filled, s) for s in (sigma_large, sigma_small)])
    az_deg = float(azimuths[0]) if isinstance(azimuths, (tuple, list)) and len(azimuths) > 0 else 315.0
    alt = np.deg2rad(ALTITUDE_DEG)
    user_range = vmin is not None and vmax is not None
    lo, hi = (max(0.0, float(vmin)), float(vmax)) if user_range else (0.0, 1.0)
    return dict(elev=elev, blurred=blurred, stats=encode_stats(elev), replace_nan=int(has_nan), nan_fill=F32(fill),
                grad_div=F32(15 * resolution / 90), az=float(np.deg2rad(az_deg)), sin_alt=float(np.sin(alt)),
                cos_alt=float(np.cos(alt)), relief=F32(relief), one_minus_relief=F32(1 - relief),
                user_range=int(user_range), vmin=F32(lo), denom=F32(hi - lo + 1e-8), vmin_is_zero=int(lo == 0.0))


def relief_contract(elev, **kw):
    """`shade` of get_relief_map(elev, None, None, None, **kw)."""
    return shade(**shade_args(elev, **kw))


def compare(got, g, parts):
    """The rule of the device's relief map against the oracle: the NaN pattern is identical; every other value is within
    TOL of `g` (the oracle's image, with its intermediates `parts` at the same pixels), except that a land pixel may
    take the adjacent colormap entry where the oracle's fp32 colormap argument x 256 lies within BOUNDARY of an integer
    (an fp32 power that rounds the other way there moves it across).  Returns (boundary pixels, worst share of TOL)."""
    assert got.shape == g.shape and got.dtype == np.float32
    assert np.array_equal(np.isnan(got), np.isnan(g))
    diff = np.nan_to_num(np.abs(got - g)).max(axis=-1)
    off = diff > TOL
    if off.any():
        arg = parts["arg"][off].astype(np.float64) * 256
        assert not parts["ocean"][off].any()
        assert np.all(np.abs(arg - np.round(arg)) <= BOUNDARY), arg[np.abs(arg - np.round(arg)) > BOUNDARY][:5]
        # the pixel is the adjacent entry across that integer, shaded with the oracle's intensity
        k = np.round(arg).astype(np.int64)
        idx = np.minimum(np.floor(arg).astype(np.int64), 255)
        alt = np.clip(np.where(idx == k, k - 1, k), 0, 255)
        alt_rgb = np.clip(LUT32[alt] * parts["gain"][off][:, None], 0, 1)
        assert float(np.abs(got[off] - alt_rgb).max()) <= TOL
    share = float(diff[~off].max()) / TOL if (~off).any() else 0.0
    return int(off.sum()), share


def worst_pixel(got, g, parts):
    """(|difference|, (row, col), whether the oracle's colormap argument there is within BOUNDARY of a LUT boundary)."""
    diff = np.nan_to_num(np.abs(got - g)).max(axis=-1)
    r, c = np.unravel_index(int(np.argmax(diff)), diff.shape)
    arg = float(parts["arg"][r, c]) * 256                 # NaN: the bad colour, no boundary
    on = np.isfinite(arg) and abs(arg - round(arg)) <= BOUNDARY and not parts["ocean"][r, c]
    return float(diff[r, c]), (int(r), int(c)), bool(on)


def mismatches(got, contract):
    """Pixels where `got` and the contract's image differ in bits (NaN == NaN) and the contract does not excuse them."""
    a, b = got.view(np.uint32), contract["rgb"].view(np.uint32)
    same = (a == b) | (np.isnan(got) & np.isnan(contract["rgb"]))
    return ~same.all(axis=-1) & ~contract["excused"]


def excuse_summary(contract) -> str:
    why, ex = contract["why"], contract["excused"]
    parts = ", ".join(f"{k} {int((v & ex).sum())}" for k, v in why.items() if (v & ex).any())
    return f"{int(ex.sum())} excused" + (f" ({parts})" if parts else "")
