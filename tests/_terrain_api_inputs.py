"""A seeded analytic world for the terrain API read-out, shared by tests/golden/make_golden_terrain_api.py (reference side)
and the terrain API tests (oracle / CUDA).  Every value is a function of the absolute pixel (i, j) through an integer
hash and exact fp64 arithmetic, so any window of it is the same on every host, and a padded window overlaps the window
it pads exactly as the pipeline's canvases do."""
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


# (scale, offset) of the five climate channels: temperature, t_season, precipitation, p_cv, lapse rate
CLIMATE = ((40.0, 12.0), (20.0, 8.0), (3000.0, 1500.0), (90.0, 50.0), (0.012, -0.006))


def planes(seed: int, i1: int, j1: int, i2: int, j2: int, specials: bool = False) -> np.ndarray:
    """fp32 [6, i2-i1, j2-j1]: elevation (metres; every 17th row x25, past the int16 clip edges) and 5 climate planes.
    With `specials`, about one elevation pixel in 18 is NaN, +inf or -inf."""
    i = np.arange(i1, i2, dtype=np.int64)[:, None] + np.zeros((1, j2 - j1), np.int64)
    j = np.arange(j1, j2, dtype=np.int64)[None, :] + np.zeros((i2 - i1, 1), np.int64)
    u = [_hash(i, j, k, seed).astype(np.float64) / 2.0 ** 32 for k in range(6)]
    elev = (u[0] - 0.5) * 3000.0 * np.where(i % 17 == 0, 25.0, 1.0)
    if specials:
        tag = _hash(i, j, 7, seed) % 54
        elev = np.where(tag == 0, np.nan, np.where(tag == 1, np.inf, np.where(tag == 2, -np.inf, elev)))
    out = [elev] + [(u[k + 1] - 0.5) * s + o for k, (s, o) in enumerate(CLIMATE)]
    return np.stack(out).astype(np.float32)


class FieldWorld:
    """What _get_terrain needs of a WorldPipeline: get(i1, j1, i2, j2, with_climate) -> {'elev', 'climate'}, CPU fp32
    tensors, over absolute pixel coordinates (negative allowed)."""

    def __init__(self, seed: int = 0, specials: bool = False):
        self.seed, self.specials = seed, specials
        self.calls = []

    def get(self, i1, j1, i2, j2, with_climate=True):
        self.calls.append((i1, j1, i2, j2))
        p = torch.from_numpy(planes(self.seed, i1, j1, i2, j2, self.specials))
        return {"elev": p[0], "climate": p[1:] if with_climate else None}


# name: (seed, specials, i1, j1, i2, j2, scale).  The torch path is picked by the padded native window: (h + w) * scale
# <= 128 takes the per-pixel-weight kernel ("small"), anything larger the separable one ("wide").
CASES = {
    "s1": (1, False, -37, 12, -25, 32, 1),
    "s2_small": (2, False, 5, -9, 21, 7, 2),
    "s2_wide": (3, False, -101, 33, -93, 193, 2),
    "s2_edge128": (4, False, 0, 0, 2, 118, 2),           # native 3 x 61: (3 + 61) * 2 = 128, still small
    "s2_edge130": (4, False, 0, 0, 2, 120, 2),           # native 3 x 62: 130, wide
    "s3": (5, False, 10, 10, 26, 31, 3),
    "s4_aligned16": (6, False, 0, 0, 16, 16, 4),
    "s8_chunk16": (7, False, -13, -29, 3, -13, 8),
    "s8_row": (8, False, 7, -300, 8, 200, 8),
    "s8_col": (9, False, -250, 3, 250, 4, 8),
    "s8_px": (10, False, -5, -5, -4, -4, 8),
    "s16_small": (11, False, 32, -48, 48, -32, 16),
    "s16_wide": (12, False, -40, 100, -20, 140, 16),
    "specials_s1": (13, True, -12, -12, 12, 12, 1),
    "specials_s2": (13, True, -12, -12, 12, 12, 2),
    "specials_s8": (14, True, -9, 3, 15, 27, 8),
}


def case_world(name):
    seed, specials, i1, j1, i2, j2, scale = CASES[name]
    return FieldWorld(seed, specials), (i1, j1, i2, j2, scale)
