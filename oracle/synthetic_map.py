"""Numpy oracle of the coarse stage's synthetic conditioning map (terrain_diffusion/inference/synthetic_map.py:182-271,
perlin_transform.py:42-45, world_pipeline.py:821-903) and of FastNoiseLite's 2-D Perlin noise with FBm fractal.

FastNoiseLite is restated from its published algorithm (FastNoiseLite.h, `_fnlGenFractalFBM2D`, `_fnlSinglePerlin2D`,
`_fnlGradCoord2D`) on fp32 arrays, with int32 arithmetic that wraps: numpy rounds every fp32 multiply and add on its
own, as a build of the library for baseline x86-64 (no FMA) does.  No value here was produced by pyfastnoiselite.
The quantile transform, `finalize`, the import merge and the signed square root follow the reference's numpy code
(NumPy >= 2: a Python scalar is rounded to the array's fp32 at each op)."""
from __future__ import annotations

import random

import numpy as np

PRIME_X = np.int32(501125321)
PRIME_Y = np.int32(1136930381)
HASH_MUL = np.int32(0x27D4EB2D)
PERLIN_SCALE = np.float32(1.4247691104677813)

# 24 unit directions at 82.5 - 15 k degrees; FastNoiseLite's 128 gradient pairs are these five times over, then the
# first 8 again
_ANGLES = np.deg2rad(82.5 - 15.0 * np.arange(24))
GRAD24 = np.stack([np.cos(_ANGLES), np.sin(_ANGLES)], axis=1).astype(np.float32)
GRADIENTS_2D = np.concatenate([np.tile(GRAD24, (5, 1)), GRAD24[:8]]).reshape(-1)        # fp32 [256]

# synthetic_map.py:219-225: (octaves, lacunarity, gain) of the five generators; the frequency is 0.05 * frequency_mult[k]
FIELD_OCTAVES = (4, 2, 4, 4, 4)
FIELD_LACUNARITY, FIELD_GAIN = 2.0, 0.5


def fast_floor(f: np.ndarray) -> np.ndarray:
    t = f.astype(np.int32)                       # C's (int)f truncates
    return np.where(f >= 0, t, t - np.int32(1)).astype(np.int32)


def lerp(a, b, t):
    return a + t * (b - a)


def interp_quintic(t):
    return t * t * t * (t * (t * np.float32(6) - np.float32(15)) + np.float32(10))


def grad_coord(seed: np.int32, xp, yp, xd, yd):
    with np.errstate(over="ignore"):
        h = (np.int32(seed) ^ xp ^ yp) * HASH_MUL
    h = h ^ (h >> np.int32(15))
    h = h & np.int32(254)
    return xd * GRADIENTS_2D[h] + yd * GRADIENTS_2D[h | 1]


def single_perlin(seed, x: np.ndarray, y: np.ndarray) -> np.ndarray:
    x0, y0 = fast_floor(x), fast_floor(y)
    xd0 = x - x0.astype(np.float32)
    yd0 = y - y0.astype(np.float32)
    xd1, yd1 = xd0 - np.float32(1), yd0 - np.float32(1)
    xs, ys = interp_quintic(xd0), interp_quintic(yd0)
    with np.errstate(over="ignore"):
        x0 = x0 * PRIME_X
        y0 = y0 * PRIME_Y
        x1, y1 = x0 + PRIME_X, y0 + PRIME_Y
    xf0 = lerp(grad_coord(seed, x0, y0, xd0, yd0), grad_coord(seed, x1, y0, xd1, yd0), xs)
    xf1 = lerp(grad_coord(seed, x0, y1, xd0, yd1), grad_coord(seed, x1, y1, xd1, yd1), xs)
    return lerp(xf0, xf1, ys) * PERLIN_SCALE


def fractal_bounding(octaves: int, gain) -> np.float32:
    g = np.abs(np.float32(gain))
    amp, frac = g, np.float32(1)
    for _ in range(1, octaves):
        frac = np.float32(frac + amp)
        amp = np.float32(amp * g)
    return np.float32(np.float32(1) / frac)


def fbm_perlin_at(seed: int, frequency, octaves: int, lacunarity, gain, x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """FastNoiseLite(seed) with NoiseType_Perlin, FractalType_FBm and these settings at fp32 coordinates (x, y):
    `gen_from_coords`.  The float settings are stored as fp32, the seed as int32 (wrapping each octave)."""
    freq, lac, gain = np.float32(frequency), np.float32(lacunarity), np.float32(gain)
    x = np.asarray(x, np.float32) * freq
    y = np.asarray(y, np.float32) * freq
    seed = np.int32((int(seed) + (1 << 31)) % (1 << 32) - (1 << 31))
    amp = fractal_bounding(octaves, gain)
    total = np.zeros_like(x)
    for _ in range(octaves):
        noise = single_perlin(seed, x, y)
        seed = np.int32((int(seed) + 1 + (1 << 31)) % (1 << 32) - (1 << 31))
        total = total + noise * amp
        # amp *= Lerp(1, ..., weighted_strength = 0) multiplies by exactly 1
        x = x * lac
        y = y * lac
        amp = np.float32(amp * gain)
    return total


def fbm_plane(seed: int, frequency, octaves: int, lacunarity, gain, i0: int, j0: int, h: int, w: int) -> np.ndarray:
    """fp32 [h, w] at x = j0 + c, y = i0 + r, the coordinates formed by np.arange(..., dtype=np.float32)."""
    xx, yy = np.meshgrid(np.arange(j0, j0 + w, dtype=np.float32), np.arange(i0, i0 + h, dtype=np.float32))
    return fbm_perlin_at(seed, frequency, octaves, lacunarity, gain, xx, yy)


def noise_seeds(seed=None) -> list:
    """The five generator seeds of make_synthetic_map_factory (synthetic_map.py:183).  Without a seed, each of the five
    draws from `random` on its own."""
    return [((seed or random.randint(0, 2 ** 30)) + k + 1) & 0x7FFFFFFF for k in range(5)]


def field_configs(frequency_mult) -> list:
    """(frequency, octaves, lacunarity, gain) of the five generators."""
    return [(0.05 * frequency_mult[k], FIELD_OCTAVES[k], FIELD_LACUNARITY, FIELD_GAIN) for k in range(5)]


def transform(noise, noise_q, data_q) -> np.ndarray:
    """transform_perlin: np.interp in fp64 with the end values outside the table."""
    return np.interp(noise, noise_q, data_q, left=data_q[0], right=data_q[-1])


def finalize(raw, stats) -> np.ndarray:
    """synthetic_map.py:232-254 on a [5, ...] raw map, in fp32."""
    a, b = float(stats["a_temp_std"]), float(stats["b_temp_std"])
    p1, p99 = float(stats["temp_std_p1"]), float(stats["temp_std_p99"])
    elev, temp, tstd, precip, pcv = (np.asarray(raw[k], np.float32) for k in range(5))
    lapse = np.clip(-6.5 + 0.0015 * precip, -9.8, -4.0) / 1000
    temp = np.clip(temp + lapse * np.maximum(0, elev), -10, 40)
    temp = np.where(temp > 20, temp, (temp - 20) * 1.25 + 20)
    t = (tstd - p1) / (p99 - p1)
    fit = a * temp + b
    baseline = np.maximum(p1, -fit)
    tstd = np.maximum(t * (p99 - baseline) + baseline + fit, 20)
    pcv = pcv * np.maximum(0, (185 - 0.04111 * precip) / 185)
    return np.stack([elev, temp, tstd, precip, pcv])


def signed_sqrt(x: np.ndarray) -> np.ndarray:
    return np.sign(x) * np.sqrt(np.abs(x))


class Factory:
    """make_synthetic_map_factory restated: __call__(i1, j1, i2, j2) -> fp32 [5, i2-i1, j2-j1] (numpy), `.sample_raw`
    (fp64, as the reference returns it) and `.finalize`.  `noise_fn(seed, frequency, octaves, lacunarity, gain, x, y) ->
    fp32` replaces the Perlin generators (the golden feeds the stand-in FastNoiseLite through it)."""

    def __init__(self, stats, frequency_mult=(1.0,) * 5, seed=None, noise_fn=None):
        self.stats = stats
        self.seeds = noise_seeds(seed)
        self.configs = field_configs(frequency_mult)
        self.noise_fn = noise_fn

    def noise(self, k, x, y):
        return (self.noise_fn or fbm_perlin_at)(self.seeds[k], *self.configs[k], x, y)

    def plane(self, k, i1, j1, i2, j2) -> np.ndarray:
        # synthetic_map.py:206-217, including its reshape of the (j2-j1, i2-i1) meshgrid to (i2-i1, j2-j1)
        xx, yy = np.meshgrid(np.arange(i1, i2, dtype=np.float32), np.arange(j1, j2, dtype=np.float32))
        v = self.noise(k, xx.ravel(), yy.ravel())
        return transform(v, self.stats[f"noise_quantiles_{k}"], self.stats[f"base_image_quantiles_{k}"]).reshape(
            i2 - i1, j2 - j1)

    def sample_raw(self, i1, j1, i2, j2) -> np.ndarray:
        return np.stack([self.plane(k, i1, j1, i2, j2) for k in range(5)])

    def finalize(self, raw) -> np.ndarray:
        return finalize(raw, self.stats)

    def __call__(self, i1, j1, i2, j2) -> np.ndarray:
        m = self.finalize(self.sample_raw(i1, j1, i2, j2))
        m[0] = signed_sqrt(m[0])
        return m


def import_override(imp, ci0, ci1, cj0, cj1):
    """world_pipeline.py:829-871 for one channel: imp = (values fp32 [rows, cols] or None, (oi, oj), default or None);
    (values, mask) or (None, None)."""
    values_in, (oi, oj), default = imp
    if values_in is None and default is None:
        return None, None
    h, w = ci1 - ci0, cj1 - cj0
    values = np.full((h, w), np.float32(0.0 if default is None else default), np.float32)
    mask = np.full((h, w), default is not None)
    if values_in is not None:
        a, b = max(ci0, oi), min(ci1, oi + values_in.shape[0])
        c, d = max(cj0, oj), min(cj1, oj + values_in.shape[1])
        if a < b and c < d:
            values[a - ci0:b - ci0, c - cj0:d - cj0] = values_in[a - oi:b - oi, c - oj:d - oj]
            mask[a - ci0:b - ci0, c - cj0:d - cj0] = True
    if not mask.any():
        return None, None
    return values, mask


def import_conditioning(factory, imports: dict, ci0, ci1, cj0, cj1) -> np.ndarray:
    """_conditioning_model_input in import mode (world_pipeline.py:873-903): the raw map of cells [ci0, ci1) x [cj0, cj1)
    (the factory's coordinates swapped) in fp32, each channel's imports merged, then the signed square root of channel
    0.  imports: {channel: (values, (oi, oj), default)}."""
    raw = np.asarray(factory.sample_raw(cj0, ci0, cj1, ci1), np.float32)
    for ch, imp in imports.items():
        values, mask = import_override(imp, ci0, ci1, cj0, cj1)
        if values is not None:
            raw[ch][mask] = values[mask]
    raw[0] = signed_sqrt(raw[0])
    return raw
