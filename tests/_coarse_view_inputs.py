"""Seeded inputs of the coarse-map and land-search cases, shared by tests/golden/make_golden_coarse_view.py (reference
side) and the coarse-view tests (oracle / CUDA).

A "world" here is what `world.coarse[:, ci0:ci1, cj0:cj1]` returns: the fp32 [7, h, w] sums (sum v*w of the six
channels, then sum w) of analytic fields on absolute coarse-cell coordinates, so a window's position matters.  Channels
0 and 1 are in signed-sqrt units, as on the coarse canvas."""
import numpy as np

LUT_SEED = 2024


def seeded_lut() -> np.ndarray:
    """fp64 [256, 3]: the stand-in for viridis' listed colours (the handler logic is pinned independently of them)."""
    return np.random.RandomState(LUT_SEED).uniform(0.0, 1.0, (256, 3))


def _analytic(seed, y, x, lo, amp):
    rng = np.random.RandomState(seed)
    out = np.zeros(y.shape)
    for _ in range(3):
        fy, fx, ph = rng.uniform(0.02, 0.3), rng.uniform(0.02, 0.3), rng.uniform(0, 6.28)
        out += rng.uniform(0.3, 1.0) * np.sin(fy * y + fx * x + ph)
    out += 0.05 * np.cos(0.71 * y * x)
    return lo + amp * out


def world_sums(kind: str, ci0: int, ci1: int, cj0: int, cj1: int) -> np.ndarray:
    """fp32 [7, h, w] sums of world `kind` over coarse cells [ci0, ci1) x [cj0, cj1)."""
    y, x = np.mgrid[ci0:ci1, cj0:cj1].astype(np.float64)
    w = 0.6 + 0.35 * np.sin(0.37 * y + 0.11 * x) * np.cos(0.23 * x)             # blended weights, never 0 here
    vals = np.stack([_analytic(31, y, x, 0.0, 25.0),                            # signed-sqrt elevation, land and sea
                     _analytic(32, y, x, 5.0, 3.0),                             # signed-sqrt p5
                     _analytic(33, y, x, 12.0, 9.0),                            # temperature
                     _analytic(34, y, x, 300.0, 150.0),                         # temperature std
                     _analytic(35, y, x, 400.0, 500.0),                         # precipitation, some below 0
                     _analytic(36, y, x, 50.0, 20.0)])                          # precipitation CV
    yy, xx = np.mgrid[ci0:ci1, cj0:cj1]
    if kind == "flat":                                                          # vmax == vmin in channels 2 and 4
        vals[2] = 7.25
        vals[4] = 130.0
    elif kind == "nan":                                                         # NaN cells, w == 0 cells, -0.0
        vals[:, (yy * 5 + xx * 3) % 13 == 0] = np.nan
        vals[3][(yy + 2 * xx) % 7 == 0] = np.nan
        w[(yy * 3 + xx) % 17 == 0] = 0.0
        vals[0][(yy - xx) % 19 == 0] = 0.0
    elif kind == "all_nan":                                                     # channels 2 and 4 entirely NaN
        vals[2] = np.nan
        vals[4] = np.nan
    elif kind == "big":                                                         # channel 3 flat at 1e17: vmin + 1 == vmin
        vals[3] = 1e17
        w[:] = 1.0
    elif kind != "mixed":
        raise KeyError(kind)
    sums = np.concatenate([vals * w, w[None]], axis=0)
    if kind == "nan":
        zero_w = (yy * 3 + xx) % 17 == 0
        odd = zero_w & ((yy + xx) % 2 == 1)
        sums[:6, odd] = vals[:, odd]                                            # v / 0 without eps: +-inf
    return sums.astype(np.float32)


# name: (world, request.args) of `coarse_png`.  Filters are `ch{c}_min` / `ch{c}_max` as the client sends them.
PNG_CASES = {
    "ch0": ("mixed", {"channel": 0, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40}),
    "ch1": ("mixed", {"channel": 1, "ci0": 3, "ci1": 40, "cj0": -30, "cj1": 11}),
    "ch2": ("mixed", {"channel": 2, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40}),
    "ch3": ("mixed", {"channel": 3, "ci0": -5, "ci1": 30, "cj0": 0, "cj1": 33}),
    "ch4_log1p": ("mixed", {"channel": 4, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40}),
    "ch5": ("mixed", {"channel": 5, "ci0": -41, "ci1": -2, "cj0": 7, "cj1": 39}),
    "defaults": ("mixed", {}),                                                   # channel 0 over [-50, 50)^2
    "flat_ch2": ("flat", {"channel": 2, "ci0": 0, "ci1": 21, "cj0": 0, "cj1": 19}),
    "flat_ch4": ("flat", {"channel": 4, "ci0": 0, "ci1": 21, "cj0": 0, "cj1": 19}),
    "nan_ch3": ("nan", {"channel": 3, "ci0": -10, "ci1": 25, "cj0": -13, "cj1": 20}),
    "nan_ch0": ("nan", {"channel": 0, "ci0": -10, "ci1": 25, "cj0": -13, "cj1": 20}),
    "all_nan_ch2": ("all_nan", {"channel": 2, "ci0": 0, "ci1": 9, "cj0": 0, "cj1": 14}),
    "all_nan_ch4": ("all_nan", {"channel": 4, "ci0": 0, "ci1": 9, "cj0": 0, "cj1": 14}),
    "big_ch3": ("big", {"channel": 3, "ci0": 0, "ci1": 9, "cj0": 0, "cj1": 14}),
    "one_cell": ("mixed", {"channel": 5, "ci0": 4, "ci1": 5, "cj0": -3, "cj1": -2}),
    "filter_lo": ("mixed", {"channel": 2, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40, "ch0_min": 0.0}),
    "filter_hi": ("mixed", {"channel": 0, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40, "ch2_max": 15.5}),
    "filter_both": ("mixed", {"channel": 4, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40, "ch3_min": 250.0,
                              "ch3_max": 420.0}),
    "filter_many": ("mixed", {"channel": 3, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40, "ch0_min": -300.0,
                              "ch2_max": 18.0, "ch4_min": 100.0, "ch5_min": 40.0, "ch5_max": 65.0}),
    "filter_ch1_ignored": ("mixed", {"channel": 2, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40, "ch1_min": 30.0,
                                     "ch1_max": 40.0}),
    "filter_ch1_and_ch5": ("mixed", {"channel": 2, "ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40, "ch1_min": 30.0,
                                     "ch5_max": 55.0}),
    "filter_nan": ("nan", {"channel": 2, "ci0": -10, "ci1": 25, "cj0": -13, "cj1": 20, "ch3_min": -1e9}),
    "filter_all_nan": ("all_nan", {"channel": 0, "ci0": 0, "ci1": 9, "cj0": 0, "cj1": 14, "ch4_max": 1e9}),
    # cells with Temp exactly 7.25 pass `<= 7.2499999` only because numpy rounds the bound to fp32 (7.25) first
    "filter_fp32_bound": ("flat", {"channel": 0, "ci0": 0, "ci1": 21, "cj0": 0, "cj1": 19, "ch2_max": 7.2499999}),
}

# name: (world, window) of `coarse_data` and `coarse_stats`
DATA_CASES = {
    "mixed": ("mixed", {"ci0": -20, "ci1": 17, "cj0": -9, "cj1": 40}),
    "nan": ("nan", {"ci0": -10, "ci1": 25, "cj0": -13, "cj1": 20}),
    "all_nan": ("all_nan", {"ci0": 0, "ci1": 9, "cj0": 0, "cj1": 14}),
    "flat": ("flat", {"ci0": 0, "ci1": 21, "cj0": 0, "cj1": 19}),
    "one_cell": ("mixed", {"ci0": 4, "ci1": 5, "cj0": -3, "cj1": -2}),
}

# (coarse_window, detail_size, min_land_frac) of `sample_land_tiles`' search; detail 256 has an empty window, 768 an
# odd tile (half 1), 1536 a window of 36 cells (a mean that is not a power-of-two fraction)
LAND_WINDOW = 24
LAND_CASES = [(LAND_WINDOW, d, f) for d in (256, 768, 1024, 1536, 8192) for f in (0.0, 0.5, 1.0)] + \
    [(LAND_WINDOW, 1024, 0.3), (LAND_WINDOW, 1024, 0.8125), (7, 1024, 0.5), (16, 8192, 0.5)]
# (seed, detail_size, min_land_frac, n_samples): random.seed(seed), then sample_land_tiles
SAMPLE_CASES = [(0, 1024, 0.5, 10), (1, 768, 0.5, 25), (2, 1536, 0.75, 3), (3, 8192, 0.5, 10000), (4, 256, 0.5, 10)]
# cells of get_coarse_climate_info in the "nan" world (w == 0 cells included)
CLIMATE_CELLS = [(0, 0), (3, -7), (1, 14), (4, 9), (-6, 2)]        # NaN, finite, w == 0 -> inf, finite, finite
