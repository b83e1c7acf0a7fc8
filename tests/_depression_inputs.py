"""Seeded elevation windows of the depression-fill and river-smoothing cases, shared by
tests/golden/make_golden_depressions.py (reference side) and the depression tests (oracle / CUDA)."""
import numpy as np

from tests._hydrology_inputs import smooth_field
from tests._post_inputs import field


def _pits():
    # smooth terrain with dug pits, NaN ocean, negative ocean and scattered NaN
    e = field(71, 72, 90, 300.0, 250.0)
    rng = np.random.RandomState(72)
    for _ in range(25):
        y, x = rng.randint(3, 69), rng.randint(3, 87)
        e[y - 2:y + 2, x - 2:x + 3] -= np.float32(rng.uniform(20, 200))
    e[e < 5] = np.nan
    e[60:72, 0:15] = -40.0
    e.flat[rng.choice(e.size, 40, replace=False)] = np.nan
    return e


def _plateau():
    # 25 m-quantised plateaus: many exact ties, flats that need the epsilon gradient; -0.0 and 0.0 ocean
    e = np.round(field(73, 64, 80, 60.0, 80.0) / np.float32(25.0)) * np.float32(25.0)
    e[40:44, 10:20] = -0.0
    e[5, 5:9] = 0.0
    return e.astype(np.float32)


def _nodata():
    e = field(74, 48, 56, 400.0, 200.0)
    e[10:14, 20:30] = -9999.0                  # <= 0: invalid in any case
    e[30:33, 5:40] = 7777.0                    # the nodata value: invalid only through `nodata`
    e[20, 20] = 7777.0
    return e


def _high():
    # elevations >= 32768 m, where fl32(m + 1e-3) == m: the epsilon add rounds away and flats stay flat
    e = np.float32(40000.0) + np.round(field(75, 40, 44, 0.0, 30.0)) * np.float32(4.0)
    e[18:22, 18:24] = 39000.0                  # a pit far below its rim
    return e.astype(np.float32)


def _inf_land():
    e = field(76, 36, 40, 200.0, 150.0)
    e[10:13, 10:30] = np.inf                   # a wall of +inf land: valid, never raised past
    e[25, 5:15] = -np.inf                      # -inf is ocean
    e[3, 3] = np.inf
    return e


def _smooth_nan():
    e = smooth_field(48, seed=77)              # NaN ocean (~1/8) for the smoothing's NaN mask
    e[0, :] = np.where(np.arange(48) % 5 == 0, np.nan, e[0, :])   # NaN on the wrapped-around edges
    e[:, -1] = np.where(np.arange(48) % 7 == 0, np.nan, e[:, -1])
    return e


# fill cases: name -> (elevation builder, keyword arguments of fill_depressions_priority_flood)
FILL_CASES = {
    "pits8": (_pits, {}),
    "pits4": (_pits, {"connectivity": 4}),
    "plateau8": (_plateau, {}),
    "plateau4": (_plateau, {"connectivity": 4}),
    "plateau_eps0": (_plateau, {"epsilon": 0.0}),
    "pits_eps005": (_pits, {"epsilon": 0.05}),
    "nodata": (_nodata, {"nodata": 7777.0}),
    "nodata4": (_nodata, {"nodata": 7777.0, "connectivity": 4}),
    "high": (_high, {}),
    "inf_land": (_inf_land, {}),
    "all_ocean": (lambda: np.minimum(field(78, 12, 16, -300.0, 100.0), np.float32(0.0)), {}),
    "row": (lambda: field(79, 1, 37, 100.0, 80.0), {}),
    "col": (lambda: field(80, 29, 1, 60.0, 70.0), {}),
    "two": (lambda: np.array([[2.0, 1.0], [1.0, 3.0]], np.float32), {}),
    "big": (lambda: smooth_field(256, seed=81), {}),
}

# smoothing cases: name -> (elevation builder, keyword arguments of smooth_river_bumps)
SMOOTH_CASES = {
    "nan": (_smooth_nan, {}),
    "iter0": (_smooth_nan, {"iterations": 0}),
    "iter1": (_smooth_nan, {"iterations": 1}),
    "params": (lambda: field(82, 40, 52, 300.0, 200.0), {"slope_thresh": 120.0, "smooth_strength": 0.2,
                                                        "iterations": 3}),
    "steep": (lambda: field(83, 33, 31, 500.0, 2000.0), {"slope_thresh": 7, "smooth_strength": 0.45}),
    "two": (lambda: np.array([[5.0, 1.0], [np.nan, 2.0]], np.float32), {}),
    "plateau": (_plateau, {}),
}


def fill_serpentine(n):
    """Adversarial n x n fill input (n even): a one-cell-wide flat channel at 100 m winds boustrophedon through
    5000 m walls, rows 1, 3, ..., n - 3, joined by one gap per wall row, alternately at the east and west end.  Its
    only outlet is the border pixel (1, 0), so every channel cell is raised by one epsilon add per cell along a single
    chain of about n^2 / 2 cells: the fill's longest dependency chain.  Returns (z, chain length)."""
    assert n % 2 == 0 and n >= 6
    z = np.full((n, n), 5000.0, np.float32)
    rows = range(1, n - 2, 2)
    for i, r in enumerate(rows):
        z[r, 1:n - 1] = 100.0
        if r + 2 < n - 2:
            z[r + 1, n - 2 if i % 2 == 0 else 1] = 100.0
    z[1, 0] = 100.0
    return z, int((z[1:-1, 1:-1] == 100.0).sum())


def fill_case(name):
    build, kw = FILL_CASES[name]
    return build(), dict(kw)


def smooth_case(name):
    build, kw = SMOOTH_CASES[name]
    return build(), dict(kw)


def composition_case():
    """The window routed after filling: plot_flow_indicator(fill_depressions_priority_flood(z))."""
    return _pits()
