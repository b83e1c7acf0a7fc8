"""TEST ORACLE (not product code): CPU restatement of the Minecraft API's read-out, terrain_diffusion/inference/
minecraft_api.py `_get_upsampled` (:265-355), `_compute_climate_vars` (:189-263), `_classify_biome` (:358-688) and
`_binary_response` (:90-99), in numpy fp32 with the reference's rounding op for op.  Only tests/ and tools may import this.
Parity: pinned bit for bit (tests/golden/minecraft_golden.npz).

- Bilinear: oracle/terrain_api.py `upsample_crop` (both of torch's CPU kernels).
- Sobel: the orders torch 2.11's CPU conv2d sums the nine exact tap products in (`sobel`), not conv2d itself.
- sqrt, asin and pow(., 1.5): torch's own CPU functions, the ones the reference calls (none is correctly rounded).
- The classifier is a per-pixel decision list (`LEAVES`, first match wins), not the reference's chain of mask writes, so
  the golden cross-checks one form against the other.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.postproc import elev_to_int16
from oracle.terrain_api import upsample_crop

F32 = np.float32


def c32(v):
    return F32(v)


# ------------------------------------------------------------------------------------------------------------ Sobel
KX = np.array([-1, 0, 1, -2, 0, 2, -1, 0, 1], F32) / F32(8)
KY = np.array([-1, -2, -1, 0, 0, 0, 1, 2, 1], F32) / F32(8)


def _sum_seq(p):
    acc = np.zeros_like(p[0])
    for v in p:
        acc = (acc + v).astype(F32)
    return acc


def _sum_pair(p):
    a = ((p[0] + p[2]).astype(F32) + (p[1] + p[3]).astype(F32)).astype(F32)
    b = ((p[4] + p[6]).astype(F32) + (p[5] + p[7]).astype(F32)).astype(F32)
    return ((a + b).astype(F32) + p[8]).astype(F32)


def _sum_one(p):
    v = [(p[j] + p[j + 4]).astype(F32) for j in range(4)]
    return (v[0] + ((v[1] + v[3]).astype(F32) + (v[2] + p[8]).astype(F32)).astype(F32)).astype(F32)


def sobel(xp: np.ndarray):
    """torch.nn.functional.conv2d(xp[None, None], sobel_{x,y}, padding=0) of the reference, bit for bit with torch 2.11's
    CPU conv2d: (dx, dy) [H, W] from xp [H+2, W+2].  Above 20480 input elements torch runs oneDNN, which sums row-major
    from 0; at or below it runs im2col + MKL gemm (K = 9), which sums blocks of 16 output pixels (flat index) as
    ((p0+p2) + (p1+p3)) + ((p4+p6) + (p5+p7)) + p8, the N % 16 tail row-major, and a single pixel as
    v_j = p_j + p_{j+4}, v0 + ((v1+v3) + (v2+p8))."""
    xp = np.asarray(xp, F32)
    H, W = xp.shape[0] - 2, xp.shape[1] - 2
    out = []
    with np.errstate(invalid="ignore", over="ignore"):
        for k in (KX, KY):
            p = [(k[a * 3 + b] * xp[a:a + H, b:b + W]).astype(F32) for a in range(3) for b in range(3)]
            seq = _sum_seq(p)
            if xp.size > 20480:
                out.append(seq)
            elif H * W == 1:
                out.append(_sum_one(p))
            else:
                n = H * W
                flat = np.arange(n).reshape(H, W)
                out.append(np.where(flat < n - n % 16, _sum_pair(p), seq).astype(F32))
    return out[0], out[1]


def gradient(xp):
    """sqrt(dx**2 + dy**2) with torch's CPU sqrt, which is not correctly rounded either."""
    dx, dy = sobel(xp)
    with np.errstate(invalid="ignore", over="ignore"):
        return _torch(torch.sqrt, ((dx * dx).astype(F32) + (dy * dy).astype(F32)).astype(F32))


def _torch(fn, x):
    return fn(torch.from_numpy(np.ascontiguousarray(x, F32))).numpy()


def _clamp(x, lo=None, hi=None):
    """torch.clamp: NaN stays NaN."""
    with np.errstate(invalid="ignore"):
        if lo is not None:
            x = np.where(np.isnan(x), x, np.maximum(x, c32(lo)))
        if hi is not None:
            x = np.where(np.isnan(x), x, np.minimum(x, c32(hi)))
    return x.astype(F32)


# ------------------------------------------------------------------------------------------------ climate variables
def climate_vars(temp, t_season, precip, p_cv) -> dict:
    """_compute_climate_vars (:208-252) in fp32, op for op (Python scalars rounded to fp32 at each op, as torch does)."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        t_std = (t_season / c32(100.0)).astype(F32)
        t_eff = _clamp((temp + (c32(0.5) * t_std).astype(F32)).astype(F32), lo=0.0)
        pet = (c32(250.0) + (c32(25.0) * t_eff).astype(F32)).astype(F32)
        pet = _clamp((pet + (c32(0.7) * (t_eff * t_eff).astype(F32)).astype(F32)).astype(F32), lo=250.0)
        aridity = (precip / _clamp(pet, lo=1.0)).astype(F32)
        penalty = (c32(1.0) - (c32(0.35) * _clamp((p_cv / c32(100.0)).astype(F32), hi=1.0)).astype(F32)).astype(F32)
        tm = (aridity * penalty).astype(F32)
        amplitude = (t_std * c32(1.414)).astype(F32)
        x = ((c32(5.0) - temp).astype(F32) / _clamp(amplitude, lo=0.1)).astype(F32)
        asin = _torch(torch.asin, _clamp(x, -1.0, 1.0))
        inner = (c32(365.0) * (c32(0.5) - (asin / c32(3.14159)).astype(F32)).astype(F32)).astype(F32)
        gs = np.where(x <= c32(-1.0), c32(365.0), np.where(x >= c32(1.0), c32(0.0), inner)).astype(F32)
        tropical = (temp >= c32(18.0)) & (t_std < c32(5.0))
    return {"tree_moisture": tm, "growing_season": gs, "tropical": tropical, "t_std": t_std}


# ------------------------------------------------------------------------------------------------------ classifier
# The decision list: (leaf name, biome id), first match wins.  Conditions are in `_leaf_conditions`.
LEAVES = (
    ("ocean_frozen", 48), ("ocean_cold", 46), ("ocean_warm", 41), ("ocean_other", 44),
    ("bare_snow", 33), ("bare", 35),
    ("mtn_snow_none", 32), ("mtn_snow_sparse", 116), ("mtn_snow_dense", 16), ("mtn_snow_noclass", 1),
    ("mtn_none_barren", 19), ("mtn_none_steppe", 31), ("mtn_none_grass", 1), ("mtn_sparse", 115), ("mtn_dense", 15),
    ("mtn_noclass", 1),
    ("snow_none", 3), ("snow_sparse", 116), ("snow_dense", 16), ("snow_noclass", 1),
    ("dry_steppe", 31), ("dry_windswept", 31), ("dry_desert", 5), ("dry_grass", 1),
    ("sf_jungle", 23), ("sf_warm_demoted", 1), ("sf_savanna", 17), ("sf_warm_forest", 108), ("sf_temperate", 108),
    ("sf_cool", 115), ("sf_frozen", 1),
    ("dense_jungle", 23), ("dense_swamp", 6), ("dense_taiga", 15), ("dense_forest", 8),
    ("rain_jungle", 23), ("rain_swamp", 6), ("rain_taiga", 15), ("rain_forest", 8),
    ("land_noclass", 1),
)
LEAF_NAMES = tuple(n for n, _ in LEAVES)
LEAF_IDS = np.array([b for _, b in LEAVES], np.int16)


def _leaf_conditions(v):
    t = v["temp"]
    frozen, hot = t < c32(-5.0), t >= c32(26.0)
    cold, cool = (t >= c32(-5.0)) & (t < c32(5.0)), (t >= c32(5.0)) & (t < c32(12.0))
    temperate, warm = (t >= c32(12.0)) & (t < c32(20.0)), (t >= c32(20.0)) & (t < c32(26.0))
    ocean, bare, mtn, snow = v["ocean"], v["slope_bare"], v["mountains"], v["has_snow"]
    none, sf, dr = v["none"], v["sparse"] | v["forest"], v["dense"] | v["rain"]
    barren, steppe, low, medium = v["barren"], v["steppe"], v["lowland"], v["slope_medium"]
    T = np.ones_like(ocean)
    return [
        ocean & frozen, ocean & cold, ocean & (warm | hot), ocean,
        bare & snow, bare,
        mtn & snow & none, mtn & snow & sf, mtn & snow & dr, mtn & snow,
        mtn & none & barren, mtn & none & steppe, mtn & none, mtn & sf, mtn & dr, mtn,
        snow & none, snow & sf, snow & dr, snow,
        none & steppe & ~barren, none & (cold | cool | temperate) & ~low & barren, none & (warm | hot), none,
        sf & hot, sf & warm & v["sparse"] & medium, sf & warm & v["sparse"], sf & warm, sf & temperate,
        sf & (cool | cold), sf,
        v["dense"] & hot, v["dense"] & warm & low, v["dense"] & (cool | cold), v["dense"],
        v["rain"] & (hot | (warm & v["tropical"])), v["rain"] & low, v["rain"] & (cool | cold), v["rain"],
        T,
    ]


def classify(elev, temp, precip, tm, gs, tropical, slope_ratio, snow_temp):
    """What _classify_biome's mask chain leaves per pixel: (biome int16 [H, W], leaf index [H, W], the variables)."""
    with np.errstate(invalid="ignore", over="ignore"):
        gs_factor = _clamp(((gs - c32(60.0)).astype(F32) / c32(90.0)).astype(F32), 0.0, 1.0)
        eff = (tm * gs_factor).astype(F32)
        mf = _clamp(((tm - c32(0.35)).astype(F32) / c32(0.45)).astype(F32), 0.0, 1.0)
        bare_t = (c32(0.7) + (c32(1.19 - 0.7) * mf).astype(F32)).astype(F32)
        sr = slope_ratio
        medium = (sr >= c32(0.62)) & (sr < bare_t)
        none0 = eff < c32(0.2)
        had_trees = ~none0 & (eff >= c32(0.5))
        alt = _clamp(elev, lo=0.0)
        v = {
            "temp": temp, "ocean": elev < c32(0.0), "slope_bare": sr >= bare_t, "slope_medium": medium,
            "mountains": alt > c32(2500.0), "lowland": alt < c32(200.0),
            "has_snow": (snow_temp < c32(0.0)) & (precip > c32(150.0)) & ~(sr > c32(0.78)),
            "none": none0, "sparse": (~none0 & (eff < c32(0.5))) | (medium & had_trees),
            "forest": ~none0 & (eff >= c32(0.5)) & (eff < c32(0.8)) & ~medium,
            "dense": ~none0 & (eff >= c32(0.8)) & (eff < c32(1.3)) & ~medium,
            "rain": ~none0 & (eff >= c32(1.3)) & ~medium,
            "barren": (tm < c32(0.05)) | (gs < c32(60.0)), "steppe": (tm < c32(0.35)) | (precip < c32(350.0)),
            "tropical": tropical, "eff": eff, "bare_threshold": bare_t, "slope_ratio": sr, "tree_moisture": tm,
            "growing_season": gs,
        }
        leaf = np.select(_leaf_conditions(v), np.arange(len(LEAVES)), default=len(LEAVES) - 1)
    return LEAF_IDS[leaf], leaf, v


# ----------------------------------------------------------------------------------------------- the whole read-out
def noise_slots(noise):
    """The reference's seven generators by the five planes that carry them: temp = snow coarse, temp = snow fine."""
    return {"temp_coarse": noise[0], "temp_fine": noise[1], "precip": noise[2], "snow_coarse": noise[0],
            "snow_fine": noise[1], "elev_coarse": noise[3], "elev_fine": noise[4]}


def readout(elev, climate, noise, scale, oi, oj, H, W, noise_scale, pixel_size_m, native_resolution, centre=None):
    """tdx_minecraft_readout's definition.  elev: [h, w] (scale >= 2: native window padded by 2; scale 1: the [H+2, W+2]
    slope window, with `centre` the [H, W] window the pixel's own elevation comes from); climate [5, ...] or None;
    noise [5, H, W].  Returns {'elev', 'elev_smooth', 'climate', 'biome', 'leaf', 'vars'}."""
    elev = np.asarray(elev, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        ring = upsample_crop(elev, scale, oi - 1, oj - 1, H + 2, W + 2)
    smooth = np.asarray(centre, F32).copy() if scale == 1 else ring[1:-1, 1:-1].copy()
    grad = gradient(ring)
    n = noise_slots(np.asarray(noise, F32))
    out_elev = smooth
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if scale > 1 and noise_scale > 0:                  # :319-351
            sf = _clamp((grad / c32(40.0 * pixel_size_m / 90.0)).astype(F32), 0.0, 1.0)
            sf = _torch(lambda t: t.pow(1.5), sf)
            amp_c = (((c32(noise_scale * 100.0) * sf).astype(F32) * c32(pixel_size_m)).astype(F32)
                     / c32(native_resolution)).astype(F32)
            amp_f = (((c32(noise_scale * 70.0) * sf).astype(F32) * c32(pixel_size_m)).astype(F32)
                     / c32(native_resolution)).astype(F32)
            d = ((n["elev_coarse"] * amp_c).astype(F32) + (n["elev_fine"] * amp_f).astype(F32)).astype(F32)
            out_elev = (smooth + (d * (smooth >= c32(0.0)).astype(F32)).astype(F32)).astype(F32)
        if climate is None:
            return {"elev": out_elev, "elev_smooth": smooth, "climate": None,
                    "biome": np.full((H, W), 1, np.int16), "leaf": None, "vars": None}
        climate = np.asarray(climate, F32)
        clim = climate.copy() if scale == 1 else upsample_crop(climate, scale, oi, oj, H, W)
        # :393-407 (numpy fp32) then :410
        temp = (clim[0] + ((c32(0.4) * n["temp_coarse"]).astype(F32) + (c32(0.2) * n["temp_fine"]).astype(F32))
                .astype(F32)).astype(F32)
        precip = (_clamp(clim[2], lo=0.0) * (c32(1.0) + (c32(0.2) * n["precip"]).astype(F32)).astype(F32)).astype(F32)
        snow = ((c32(3.0) * n["snow_coarse"]).astype(F32) + (c32(2.0) * n["snow_fine"]).astype(F32)).astype(F32)
        cv = climate_vars(temp, clim[1], precip, clim[3])
        sr = (grad / c32(pixel_size_m)).astype(F32)
        biome, leaf, v = classify(smooth, temp, precip, cv["tree_moisture"], cv["growing_season"], cv["tropical"], sr,
                                  (temp + snow).astype(F32))
    v["gradient"] = grad
    return {"elev": out_elev, "elev_smooth": smooth, "climate": clim, "biome": biome, "leaf": leaf, "vars": v}


def minecraft_window(i1: int, j1: int, i2: int, j2: int, scale: int):
    """The windows the handlers read: scale 1 (_handle_1x :714-727) -> the slope window (i1-1, j1-1, i2+1, j2+1) with
    the crop at (1, 1); scale >= 2 (_get_upsampled :272-307) -> the native window padded by 2 and the crop origin in its
    upsampled version.  (wi1, wj1, wi2, wj2, oi, oj); Python floor / ceil division."""
    if scale == 1:
        return i1 - 1, j1 - 1, i2 + 1, j2 + 1, 1, 1
    ni1, nj1 = i1 // scale, j1 // scale
    ni2, nj2 = -(-i2 // scale), -(-j2 // scale)
    return ni1 - 2, nj1 - 2, ni2 + 2, nj2 + 2, 2 * scale + i1 - ni1 * scale, 2 * scale + j1 - nj1 * scale


def request(get, i1, j1, i2, j2, scale, noise_scale, native_resolution, noise_planes):
    """A whole `/terrain` request on `get(i1, j1, i2, j2, with_climate)` (numpy fp32 planes), with
    `noise_planes(i1, j1, H, W)` -> [5, H, W]: the dict of `readout` plus the wire body."""
    H, W = i2 - i1, j2 - j1
    wi1, wj1, wi2, wj2, oi, oj = minecraft_window(i1, j1, i2, j2, scale)
    if scale == 1:
        slope = get(wi1, wj1, wi2, wj2, False)["elev"]
        out = get(i1, j1, i2, j2, True)
        r = readout(slope, out["climate"], noise_planes(i1, j1, H, W), 1, 1, 1, H, W, noise_scale,
                    native_resolution, native_resolution, centre=out["elev"])
    else:
        out = get(wi1, wj1, wi2, wj2, True)
        r = readout(out["elev"], out["climate"], noise_planes(i1, j1, H, W), scale, oi, oj, H, W, noise_scale,
                    native_resolution / scale, native_resolution)
    r["body"] = payload(r["elev"], r["biome"])
    return r


def payload(elev, biome) -> bytes:
    """_binary_response's body: int16-LE elevation (floor, clip; NaN -> 0), then int16-LE biome ids."""
    return elev_to_int16(elev).tobytes() + np.asarray(biome).astype("<i2").tobytes()
