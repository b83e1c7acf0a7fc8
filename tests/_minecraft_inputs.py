"""Inputs for the Minecraft API read-out, shared by tests/golden/make_golden_minecraft.py (reference side) and the
Minecraft API tests (oracle / CUDA).

- `FastNoiseLite`: a stand-in with pyfastnoiselite's attribute surface (constructor seed, noise_type, frequency,
  fractal_type / _octaves / _lacunarity / _gain, gen_from_coords(coords [2, N] fp32) -> fp32 [N]).  It is not Perlin
  noise: its value is a deterministic function in [-1, 1] of the coordinates and of every configuration field, so equal
  configurations agree and different ones differ.  `install_stand_in()` puts it in sys.modules as
  `pyfastnoiselite.pyfastnoiselite`, where the reference (and the product's default noise provider) import it from.
- `BiomeWorld`: an analytic world whose `get()` slices planes on absolute pixel coordinates, like
  tests/_terrain_api_inputs.FieldWorld.  Its planes cover the classifier's cross product: temperature -25..35 C,
  seasonality 0..1500, precipitation 0..4000 mm, ocean of every temperature band (with steep floors), land above 2500 m,
  ramps and cliffs steep enough for slope_medium and slope_bare at every scale, and NaN climate pixels.
"""
import enum
import math
import sys
import types

import numpy as np
import torch

M32 = 0xFFFFFFFF


def _hash(i, j, k, seed):
    v = (i * 0x9E3779B1 + j * 0x85EBCA77 + k * 0xC2B2AE3D + seed * 0x27D4EB2F) & M32
    v ^= v >> 15
    v = (v * 0x2C1B3C6D) & M32
    v ^= v >> 12
    v = (v * 0x297A2D39) & M32
    return v ^ (v >> 15)


# ----------------------------------------------------------------------------------------------- FastNoiseLite stand-in
class NoiseType(enum.IntEnum):
    NoiseType_OpenSimplex2 = 0
    NoiseType_Perlin = 3


class FractalType(enum.IntEnum):
    FractalType_None = 0
    FractalType_FBm = 1


class FastNoiseLite:
    def __init__(self, seed: int = 1337):
        self.seed = seed
        self.noise_type = NoiseType.NoiseType_OpenSimplex2
        self.frequency = 0.01
        self.fractal_type = FractalType.FractalType_None
        self.fractal_octaves = 3
        self.fractal_lacunarity = 2.0
        self.fractal_gain = 0.5

    def _key(self):
        return (int(self.seed), int(self.noise_type), float(np.float32(self.frequency)), int(self.fractal_type),
                int(self.fractal_octaves), float(np.float32(self.fractal_lacunarity)),
                float(np.float32(self.fractal_gain)))

    def gen_from_coords(self, coords) -> np.ndarray:
        coords = np.asarray(coords, np.float32)
        assert coords.ndim == 2 and coords.shape[0] == 2
        key = self._key()
        h = 0
        for v in key:
            h = _hash(h, int(round(v * 1e6)) & M32, 17, 3)
        x, y = coords[0].astype(np.float64), coords[1].astype(np.float64)
        f, amp, total, norm = key[2], 1.0, 0.0, 0.0
        for o in range(max(1, key[4])):
            a = (_hash(h, o, 1, 5) / 2.0 ** 32) * 2 * math.pi
            ph = (_hash(h, o, 2, 7) / 2.0 ** 32) * 2 * math.pi
            total = total + amp * np.sin(f * (x * math.cos(a) + y * math.sin(a)) * 6.0 + ph)
            norm += amp
            f *= key[5]
            amp *= key[6]
        # a per-pixel hash term keeps neighbouring pixels distinct even at low frequencies
        ix, iy = coords[0].astype(np.int64), coords[1].astype(np.int64)
        jitter = (_hash(ix, iy, 11, h & 0xFFFF) / 2.0 ** 32 - 0.5) * 0.2
        return np.clip(total / norm * 0.9 + jitter, -1.0, 1.0).astype(np.float32)


def install_stand_in() -> types.ModuleType:
    """Put the stand-in where `from pyfastnoiselite.pyfastnoiselite import FastNoiseLite, NoiseType, FractalType` finds
    it; returns the inner module."""
    inner = types.ModuleType("pyfastnoiselite.pyfastnoiselite")
    inner.FastNoiseLite, inner.NoiseType, inner.FractalType = FastNoiseLite, NoiseType, FractalType
    outer = types.ModuleType("pyfastnoiselite")
    outer.pyfastnoiselite = inner
    sys.modules["pyfastnoiselite"], sys.modules["pyfastnoiselite.pyfastnoiselite"] = outer, inner
    return inner


def stand_in_noise(cfg, i0: int, j0: int, h: int, w: int) -> np.ndarray:
    """A `noise_fn` over the stand-in: the generator of configuration `cfg` at x = j0 + c, y = i0 + r."""
    g = FastNoiseLite(seed=cfg.seed)
    g.noise_type = NoiseType.NoiseType_Perlin
    g.frequency = cfg.frequency
    g.fractal_type = FractalType.FractalType_FBm
    g.fractal_octaves = cfg.octaves
    g.fractal_lacunarity = cfg.lacunarity
    g.fractal_gain = cfg.gain
    xx, yy = np.meshgrid(np.arange(j0, j0 + w, dtype=np.float32), np.arange(i0, i0 + h, dtype=np.float32))
    return g.gen_from_coords(np.array([xx.ravel(), yy.ravel()], np.float32)).reshape(h, w)


# ------------------------------------------------------------------------------------------------------- the world
CELL = 9                       # native pixels per elevation cell


def planes(seed: int, i1: int, j1: int, i2: int, j2: int) -> np.ndarray:
    """fp32 [6, i2-i1, j2-j1]: elevation (metres) and 5 climate planes (temperature C, seasonality, precipitation mm,
    precipitation CV %, lapse rate), functions of the absolute native pixel."""
    i = np.arange(i1, i2, dtype=np.int64)[:, None] + np.zeros((1, j2 - j1), np.int64)
    j = np.arange(j1, j2, dtype=np.int64)[None, :] + np.zeros((i2 - i1, 1), np.int64)
    u = [_hash(i, j, k, seed).astype(np.float64) / 2.0 ** 32 for k in range(8)]
    ci, cj = np.floor_divide(i, CELL), np.floor_divide(j, CELL)
    cu = [_hash(ci, cj, 20 + k, seed).astype(np.float64) / 2.0 ** 32 for k in range(4)]
    # cell kind: ocean 30 %, lowland 25 %, midland 20 %, mountain 25 %; within a cell: flat, ramp or cliff
    base = np.select([cu[0] < 0.3, cu[0] < 0.55, cu[0] < 0.75], [-20.0 - 1500.0 * cu[1], 5.0 + 180.0 * cu[1],
                                                                 300.0 + 2000.0 * cu[1]], 2700.0 + 1500.0 * cu[1])
    texture = np.select([cu[2] < 0.45, cu[2] < 0.8],
                        [(u[0] - 0.5) * 20.0,                                          # flat
                         (np.mod(i, CELL) * np.cos(6.3 * cu[3]) + np.mod(j, CELL) * np.sin(6.3 * cu[3]))
                         * (40.0 + 110.0 * cu[3])],                                    # ramp: 40..150 m / pixel
                        (u[0] - 0.5) * 400.0)                                          # cliff
    elev = base + texture
    elev = np.where(base < 0, np.minimum(elev, -1.0), elev)                            # ocean cells stay ocean
    temp = -25.0 + 60.0 * u[2]
    t_season = 1500.0 * u[3]
    precip = 4000.0 * u[4] ** 2
    p_cv = 150.0 * u[5]
    # snowy ramps: land at 500 m rising 68.4 m per pixel (slope ratio 0.76 at 90 m) in a cold, just-wet-enough climate,
    # so that the moisture-dependent bare threshold falls below the 0.78 snow cut-off (bare rock that keeps its snow)
    snowy = cu[2] >= 0.93
    elev = np.where(snowy, 500.0 + np.mod(i, CELL) * 68.4, elev)
    temp = np.where(snowy, -12.0 + 4.0 * u[2], temp)
    t_season = np.where(snowy, 300.0, t_season)
    precip = np.where(snowy, 165.0, precip)
    p_cv = np.where(snowy, 100.0, p_cv)
    lapse = (u[6] - 0.5) * 0.012
    tag = _hash(i, j, 31, seed) % 97                                                    # NaN climate pixels
    temp = np.where(tag == 0, np.nan, temp)
    precip = np.where(tag == 1, np.nan, precip)
    p_cv = np.where(tag == 2, np.nan, p_cv)
    t_season = np.where(tag == 3, np.nan, t_season)
    return np.stack([elev, temp, t_season, precip, p_cv, lapse]).astype(np.float32)


class BiomeWorld:
    """What the Minecraft handlers need of a WorldPipeline: get(i1, j1, i2, j2, with_climate) -> {'elev', 'climate'}
    (CPU fp32 tensors, absolute coordinates, negative allowed) and native_resolution."""

    def __init__(self, seed: int = 0, native_resolution: float = 90.0):
        self.seed, self.native_resolution = seed, native_resolution
        self.calls = []

    def get(self, i1, j1, i2, j2, with_climate=True):
        self.calls.append((i1, j1, i2, j2, with_climate))
        p = torch.from_numpy(planes(self.seed, i1, j1, i2, j2))
        return {"elev": p[0], "climate": p[1:] if with_climate else None}

    def get_np(self, i1, j1, i2, j2, with_climate=True):
        out = self.get(i1, j1, i2, j2, with_climate)
        return {k: (None if v is None else v.numpy()) for k, v in out.items()}


# name: (seed, native_resolution, i1, j1, i2, j2, scale, noise).  Scale 1 reads the window and its 1-pixel ring; scale
# s >= 2 the native window padded by 2, whose upsampled size picks torch's bilinear kernel: (h + w) * s <= 128 is the
# per-pixel-weight kernel.  The "switch" cases are small by the unpadded or 1-padded window and wide by the 2-padded one.
# The golden file stores, for every case, a digest of the response body (int16 elevation + biome ids) and of each
# output array; the body only for windows of at most BODY_LIMIT pixels and the arrays only for windows of at most
# FULL_LIMIT pixels, which keeps the file small.
CASES = {
    "s1_200x300": (1, 90.0, -120, 40, 80, 340, 1, 1.0),
    "s1_px": (2, 90.0, 5, -7, 6, -6, 1, 1.0),
    "s1_row": (3, 90.0, -3, -250, -2, 250, 1, 0.0),
    "s1_16_nr30": (4, 30.0, -8, -8, 8, 8, 1, 1.0),
    "s2_64x96": (5, 90.0, -40, -60, 24, 36, 2, 1.0),
    "s2_col": (6, 90.0, 10, 3, 210, 4, 2, -1.0),
    "s2_16_nr30": (7, 30.0, 0, 0, 16, 16, 2, 1.0),
    "s2_switch": (8, 90.0, 0, 0, 16, 100, 2, 1.0),
    "s2_100x150": (9, 90.0, -51, 77, 49, 227, 2, 1.0),
    "s4_16": (10, 90.0, -37, 21, -21, 37, 4, 1.0),
    "s4_switch": (11, 90.0, 0, 0, 40, 64, 4, 1.0),
    "s4_64x96_noise0": (12, 90.0, -1000, 500, -936, 596, 4, 0.0),
    "s8_16": (13, 90.0, -13, -29, 3, -13, 8, 1.0),
    "s8_px": (14, 90.0, -5, -5, -4, -4, 8, 1.0),
    "s8_200x300_nr30": (15, 30.0, 400, -1200, 600, -900, 8, 1.0),
    "s8_row_noise_neg": (16, 90.0, 7, -300, 8, 200, 8, -1.0),
    "s16_16": (17, 90.0, 32, -48, 48, -32, 16, 1.0),
    "s16_64x96": (18, 90.0, -2000, -3000, -1936, -2904, 16, 1.0),
}


FULL_LIMIT = 2600
BODY_LIMIT = 20000


def digest(a) -> str:
    """SHA-256 of an output array's shape, dtype and little-endian bytes, every NaN written as 0x7FC00000 (a NaN's sign
    and payload are the producer's)."""
    import hashlib
    a = np.ascontiguousarray(a)
    if a.dtype == np.float32:
        a = np.where(np.isnan(a), np.float32(np.nan), a).astype("<f4")
        a = np.where(np.isnan(a), np.uint32(0x7FC00000), a.view(np.uint32)).astype("<u4")
    h = hashlib.sha256(f"{a.shape}{a.dtype.str}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def case_world(name):
    seed, nr, i1, j1, i2, j2, scale, noise = CASES[name]
    return BiomeWorld(seed, nr), (i1, j1, i2, j2, scale, noise)
