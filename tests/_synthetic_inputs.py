"""Inputs for the synthetic conditioning map, shared by tests/golden/make_golden_synthetic.py (reference side) and the
synthetic-map tests (oracle / CUDA).

- `stats_fixture()`: seeded statistics in the reference's JSON cache format (`data/global/synthetic_map_stats.json`,
  synthetic_map.py:159-180): five strictly increasing 64-knot noise-quantile tables over the range FBm noise covers and
  five data tables in the units of the WorldClim / ETOPO channels (elevation m, temperature C, temperature-std residual,
  precipitation mm, precipitation CV %), plus a temperature-std fit and its 0.1 / 99.9 percentiles.  The even knots of
  every noise table and its last knot are fp32 values (so fp32 noise can land exactly on them), the other odd knots
  arbitrary doubles.
- `CASES`: factory windows (i1, j1, i2, j2) with the seed and `frequency_mult` they are drawn with: negative windows,
  windows straddling 0 and +-2^24 (where np.arange's fp32 coordinates stop being exact), non-square windows (the
  reference's reshape reinterprets them), and seeds 0 / None (drawn from `random` after `random.seed(draw)`), 2^31 - 1,
  above 2^32 and 2^64 - 1.
- `knot_noise()`: a [5, 8, 16] noise stack per channel below, above, exactly on and between the table's knots.
- `knot_raw()`: a [5, 8, 16] raw map across every branch of `finalize`.
- `IMPORT_CASES`: square windows (the coarse stage's are 64^2) with imported rasters that overlap them partly, cover them, miss
  them, carry NaN and -0.0, and with or without a default value.
"""
from __future__ import annotations

import json

import numpy as np

N_KNOTS = 64


def _table(rng, lo, hi, fp32_even: bool) -> list:
    q = np.sort(rng.uniform(0.0, 1.0, N_KNOTS))
    q = lo + (hi - lo) * (q - q[0]) / (q[-1] - q[0])
    q = np.maximum.accumulate(q + np.arange(N_KNOTS) * 1e-6 * (hi - lo))   # strictly increasing
    if fp32_even:
        q[::2] = q[::2].astype(np.float32).astype(np.float64)
        q[-1] = np.float64(np.float32(q[-1]))
    assert np.all(np.diff(q) > 0)
    return q.tolist()


# data ranges per channel: elevation (m), temperature (C), temperature std residual, precipitation (mm), precip CV (%)
DATA_RANGES = [(-6500.0, 6200.0), (-25.0, 31.0), (-520.0, 760.0), (0.0, 7800.0), (4.0, 160.0)]


def stats_fixture(seed: int = 20261017) -> dict:
    """The cache's JSON payload (plain lists and floats)."""
    rng = np.random.default_rng(seed)
    noise = [_table(rng, -0.62 + 0.01 * k, 0.58 - 0.01 * k, True) for k in range(5)]
    data = [_table(rng, lo, hi, False) for lo, hi in DATA_RANGES]
    return {"n_quantiles": N_KNOTS, "noise_quantile_tables": noise, "data_quantile_tables": data,
            "a_temp_std": -24.871339271940734, "b_temp_std": 1016.3345192834561,
            "temp_std_p1": -402.4166259765625 + 0.123456789, "temp_std_p99": 689.0712890625 - 0.987654321}


def stats_mapping(payload: dict | None = None) -> dict:
    """The reference's in-memory form of a payload (synthetic_map.py:134-157)."""
    payload = stats_fixture() if payload is None else payload
    stats = {k: float(payload[k]) for k in ("a_temp_std", "b_temp_std", "temp_std_p1", "temp_std_p99")}
    for k, t in enumerate(payload["noise_quantile_tables"]):
        stats[f"noise_quantiles_{k}"] = np.asarray(t, np.float64)
    for k, t in enumerate(payload["data_quantile_tables"]):
        stats[f"base_image_quantiles_{k}"] = np.asarray(t, np.float64)
    return stats


def write_stats(path, payload: dict | None = None) -> None:
    with open(path, "w", encoding="utf-8") as f:
        json.dump(stats_fixture() if payload is None else payload, f)


FREQ_SYNTH = [1.5, 3, 3, 3, 3]       # WorldPipeline's default frequency_mult
FREQ_ONES = [1.0] * 5                # make_synthetic_map_factory's default
BIG = 1 << 24

# name: (seed, draw, frequency_mult, (i1, j1, i2, j2)); `draw` seeds `random` before the factory is made (it matters
# for seed 0 and None only)
CASES = {
    "neg": (12345, 0, FREQ_SYNTH, (-200, -150, -168, -118)),
    "zero": (0, 1, FREQ_SYNTH, (-20, -30, 12, 2)),
    "none": (None, 2, FREQ_ONES, (-31, 17, 1, 49)),
    "int31": ((1 << 31) - 1, 3, FREQ_SYNTH, (100, -32, 132, 0)),
    "above32": ((1 << 32) + 77, 4, FREQ_ONES, (-7, -9, 25, 23)),
    "u64max": ((1 << 64) - 1, 5, FREQ_SYNTH, (3, 5, 35, 37)),
    "big_i": (99, 6, FREQ_SYNTH, (BIG - 16, -20, BIG + 16, 12)),
    "big_neg": (4242, 7, FREQ_ONES, (-20, -BIG - 16, 12, -BIG + 16)),
    "big_both": (7, 8, FREQ_SYNTH, (3 * BIG - 5, -2 * BIG - 20, 3 * BIG + 27, -2 * BIG + 12)),
    "wide": (31337, 9, FREQ_SYNTH, (5, -7, 45, 17)),
    "tall": (31338, 10, FREQ_ONES, (-12, 40, 4, 101)),
    "row": (555, 11, FREQ_SYNTH, (-40, 9, 23, 10)),
}


def knot_noise(payload: dict | None = None) -> np.ndarray:
    """fp32 [5, 8, 16]: per channel, noise below the table, above it, exactly on every even knot, next to the odd
    knots (their fp32 rounding), at the end knots, and between knots."""
    payload = stats_fixture() if payload is None else payload
    out = np.empty((5, 8 * 16), np.float32)
    rng = np.random.default_rng(7)
    for k, t in enumerate(payload["noise_quantile_tables"]):
        t = np.asarray(t)
        vals = [t[0] - 0.25, t[0] - 1e-6, t[-1] + 1e-6, t[-1] + 0.3, t[0], t[-1], -1.0, 1.0, 0.0, -0.0]
        vals += t[::2].tolist() + t[1::2].tolist()                      # on / next to every knot
        vals += (0.5 * (t[:-1] + t[1:]))[:128 - len(vals) - 10].tolist()
        vals += rng.uniform(t[0], t[-1], 128 - len(vals)).tolist()
        out[k] = np.asarray(vals, np.float64).astype(np.float32)
    return out.reshape(5, 8, 16)


def knot_raw() -> np.ndarray:
    """fp32 [5, 8, 16] raw maps for `finalize` alone: values across every clip, the 20 C pivot, the 185 mm cut and
    both zero signs."""
    rng = np.random.default_rng(11)
    elev = np.concatenate([[0.0, -0.0, 1.0, -1.0, 8000.0, -8000.0], rng.uniform(-7000, 7000, 122)])
    temp = np.concatenate([[20.0, 20.0000019, 19.999998, -10.0, 40.0, 45.0, -30.0, 0.0], rng.uniform(-30, 45, 120)])
    tstd = np.concatenate([[-402.0, 689.0, 0.0, -0.0], rng.uniform(-700, 900, 124)])
    precip = np.concatenate([[0.0, 185.0 / 0.04111, 4500.0, 6000.0, -0.0, 1.0], rng.uniform(0, 9000, 122)])
    pcv = np.concatenate([[0.0, -0.0, 200.0], rng.uniform(0, 180, 125)])
    return np.stack([elev, temp, tstd, precip, pcv]).astype(np.float32).reshape(5, 8, 16)


def _raster(seed, rows, cols, lo, hi, specials=True) -> np.ndarray:
    rng = np.random.default_rng(seed)
    v = rng.uniform(lo, hi, (rows, cols)).astype(np.float32)
    if specials:
        v.flat[::17] = np.nan
        v.flat[5::23] = -0.0
        v.flat[9::29] = 0.0
    return v


# name: ((ci0, ci1, cj0, cj1) square window, factory case providing seed / frequency_mult,
#        {channel: (values | None, (oi, oj), default | None)})
IMPORT_CASES = {
    "partial": ((-48, -16, 0, 32), "neg", {
        0: (_raster(1, 40, 30, -3000.0, 4000.0), (-60, 20), None),
        3: (_raster(2, 100, 100, 0.0, 3000.0), (-30, -50), None),
    }),
    "defaults": ((48, 80, -96, -64), "int31", {
        1: (_raster(3, 20, 200, -10.0, 30.0), (60, -150), 12.5),
        2: (_raster(10, 2, 2, 0.0, 50.0), (5000, 5000), -0.0),          # only the default reaches it
        4: (_raster(4, 10, 10, 0.0, 100.0), (1000, 1000), None),     # misses the window: no override
    }),
    "cover_all": ((-2, 30, -3, 29), "zero", {
        0: (_raster(5, 80, 80, -100.0, 100.0), (-10, -10), 1.0),
        1: (_raster(6, 32, 32, -5.0, 5.0), (-2, -3), None),
        2: (_raster(11, 5, 5, 0.0, 50.0), (20, 20), 300.0),
        3: (_raster(7, 3, 70, 100.0, 900.0), (10, -5), float("nan")),
        4: (_raster(8, 64, 1, 10.0, 90.0), (-2, 20), None),
    }),
    "big": ((BIG - 16, BIG + 16, -BIG - 16, -BIG + 16), "big_both", {
        0: (_raster(9, 50, 50, -500.0, 500.0), (BIG - 40, -BIG), -0.0),
    }),
}


def stand_in_fields(seed, frequency, octaves, lacunarity, gain, x, y) -> np.ndarray:
    """The stand-in FastNoiseLite of tests/_minecraft_inputs.py configured as the reference's factory configures its
    generators, at fp32 coordinates (x, y): the `noise_fn` of oracle/synthetic_map.Factory that reproduces the golden."""
    from tests._minecraft_inputs import FastNoiseLite, FractalType, NoiseType
    g = FastNoiseLite(seed=seed)
    g.noise_type = NoiseType.NoiseType_Perlin
    g.frequency = frequency
    g.fractal_type = FractalType.FractalType_FBm
    g.fractal_octaves = octaves
    g.fractal_lacunarity = lacunarity
    g.fractal_gain = gain
    return g.gen_from_coords(np.array([np.ravel(x), np.ravel(y)], np.float32)).reshape(np.shape(x))
