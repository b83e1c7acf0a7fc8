"""Seeded inputs of the explorer detail-view cases, shared by tests/golden/make_golden_explorer.py (reference side) and
the explorer tests (oracle / CUDA).

A "world" here is what the handlers' `world.get(i1, j1, i2, j2)` returns: analytic fp32 planes on absolute pixel
coordinates (so a window's position matters), elevation with land and ocean and climate plane 0 a temperature."""
import numpy as np

NATIVE_RESOLUTION = 30.0


def _analytic(seed, i1, j1, i2, j2, lo, amp):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[i1:i2, j1:j2].astype(np.float64)
    out = np.zeros(y.shape)
    for _ in range(4):
        fy, fx, ph = rng.uniform(0.005, 0.08), rng.uniform(0.005, 0.08), rng.uniform(0, 6.28)
        out += rng.uniform(0.3, 1.0) * np.sin(fy * y + fx * x + ph)
    out += 0.01 * np.cos(0.37 * y * x)                           # a little high-frequency detail, still on coordinates
    return lo + amp * out


def world_planes(kind: str, i1: int, j1: int, i2: int, j2: int):
    """(elev fp32 [H, W], climate fp32 [5, H, W]) of world `kind` over rows [i1, i2) x columns [j1, j2)."""
    elev = _analytic(11, i1, j1, i2, j2, 200.0, 900.0)
    temp = 15.0 - np.maximum(elev, 0.0) / 150.0 + _analytic(12, i1, j1, i2, j2, 0.0, 4.0)
    climate = np.stack([temp] + [_analytic(13 + c, i1, j1, i2, j2, 10.0 * c, 5.0) for c in range(4)])
    y, x = np.mgrid[i1:i2, j1:j2]
    if kind == "flat":                                          # vmax == vmin: the +1 fix
        elev, climate[0] = np.full_like(elev, 850.0), np.full_like(elev, -3.25)
    elif kind == "nan_temp":
        climate[0][(y * 7 + x * 3) % 11 == 0] = np.nan
    elif kind == "nan_relief":                                  # NaN on land, a positive NaN-median: transparent pixels
        elev = np.abs(elev) + 50.0
        elev[((y - i1) // 4 + (x - j1) // 5) % 7 == 0] = np.nan
    elif kind == "specials":                                    # raw body: NaN, +-inf, beyond int16, -0.5, -0.0
        e = elev.reshape(-1)
        e[:8] = (np.nan, np.inf, -np.inf, 40000.0, -40000.0, -0.5, -0.0, 32767.9)
        e[8:12] = (-32768.0, -32768.5, 0.99, -1e-30)
        t = climate[0].reshape(-1)
        t[:4] = (np.nan, np.inf, -np.inf, -0.0)
    elif kind != "mixed":
        raise KeyError(kind)
    return elev.astype(np.float32), climate.astype(np.float32)


# name: (world, endpoint, request.args).  The endpoint is 'png' (detail_png) or 'raw' (detail_raw).
HANDLER_CASES = {
    "elevation": ("mixed", "png", {"mode": "elevation", "ci": 1, "cj": -1, "detail_size": 64}),
    "temperature": ("mixed", "png", {"mode": "temperature", "ci": 1, "cj": -1, "detail_size": 64}),
    "relief": ("mixed", "png", {"ci": 1, "cj": -1, "detail_size": 64}),                # mode defaults to 'relief'
    "unknown_mode": ("mixed", "png", {"mode": "biome", "ci": 0, "cj": 2, "detail_size": 40}),   # the else branch
    "odd_elevation": ("mixed", "png", {"mode": "elevation", "ci": -2, "cj": -3, "detail_size": 33, "pan_i": -7,
                                       "pan_j": 5}),
    "odd_temperature": ("mixed", "png", {"mode": "temperature", "ci": -1, "cj": 0, "detail_size": 47, "pan_i": 130,
                                         "pan_j": -301}),
    "odd_relief": ("mixed", "png", {"ci": -1, "cj": -1, "detail_size": 35, "pan_i": -3, "pan_j": -200}),
    "flat_elevation": ("flat", "png", {"mode": "elevation", "detail_size": 24}),
    "flat_temperature": ("flat", "png", {"mode": "temperature", "detail_size": 24}),
    "nan_temperature": ("nan_temp", "png", {"mode": "temperature", "ci": 3, "detail_size": 48}),
    "nan_relief": ("nan_relief", "png", {"ci": 2, "cj": 1, "detail_size": 48}),
    "raw": ("mixed", "raw", {"ci": 1, "cj": -1, "detail_size": 64}),
    "raw_odd": ("mixed", "raw", {"ci": -1, "cj": 0, "detail_size": 47, "pan_i": 130, "pan_j": -301}),
    "raw_specials": ("specials", "raw", {"ci": 0, "cj": 0, "detail_size": 20, "pan_i": 10, "pan_j": 10}),
}


def _big():
    p = np.full((6, 7), 1e17, np.float32)
    p[2, 3] = p[4, 0] = np.nan
    return p


def _ramp(n=64):
    return np.linspace(-3.0, 5.0, n * n, dtype=np.float32).reshape(n, n)


def _with(p, idx, vals):
    p = p.copy()
    p.flat[list(idx)] = vals
    return p


def _field(seed, h, w, lo=300.0, amp=500.0):
    return _analytic(seed, 0, 0, h, w, lo, amp).astype(np.float32)


# name: (plane builder, colormap).  Planes get() does not produce; they go through the handler with a world whose
# get() returns the plane as the elevation (terrain) or the temperature (RdBu_r).
PLANE_CASES = {
    "all_nan": (lambda: np.full((7, 9), np.nan, np.float32), "terrain"),
    "big_terrain": (_big, "terrain"),                              # vmin + 1 == vmin: everything colour 0, NaN included
    "big_rdbu": (_big, "RdBu_r"),
    "ramp_terrain": (_ramp, "terrain"),                            # every table entry, x * 256 == 256 at the top
    "ramp_rdbu": (_ramp, "RdBu_r"),
    "pos_inf": (lambda: _with(_field(21, 9, 11), (5, 40), (np.inf, np.nan)), "terrain"),
    "neg_inf": (lambda: _with(_field(22, 9, 11), (3,), (-np.inf,)), "RdBu_r"),
    "both_inf": (lambda: _with(_field(23, 5, 6), (0, 29), (np.inf, -np.inf)), "terrain"),
    # the middle value takes table entry 168 with Normalize's fp64 steps and 167 with fp32 arithmetic throughout
    "nep50": (lambda: np.array([[-1728.9300537109375, 1161.9034423828125, 2249.851806640625]], np.float32), "terrain"),
    "one_by_one": (lambda: np.array([[42.0]], np.float32), "terrain"),
    "one_by_n": (lambda: _field(24, 1, 37), "RdBu_r"),
    "n_by_one": (lambda: _field(25, 29, 1, -5.0, 20.0), "terrain"),
}


def plane_case(name):
    build, cmap = PLANE_CASES[name]
    return build(), cmap
