"""Seeded elevation windows of the shaded-relief cases, shared by tests/golden/make_golden_relief.py (reference side)
and the relief tests (oracle / CUDA)."""
import numpy as np

from tests._post_inputs import field


def _nan_case():
    e = field(43, 64, 48, -400.0, 300.0)
    rng = np.random.RandomState(44)
    e.flat[rng.choice(e.size, 150, replace=False)] = np.nan       # 2922 finite values: the median is a mean of two
    e[10:14, 20:30] = np.nan
    return e


CASES = {
    # name: (elevation builder, get_relief_map keyword arguments)
    "mixed": (lambda: field(41, 256, 320, 300.0, 600.0), {}),                               # land + ocean, vmin == 0
    "land": (lambda: field(42, 200, 176, 2000.0, 300.0), {"resolution": 30, "relief": 0.7}),  # hero-figure arguments
    "nan": (_nan_case, {}),
    "tiny": (lambda: field(45, 5, 7, 100.0, 50.0), {}),                                       # filters reflect often
    "flat": (lambda: np.full((40, 56), 850.0, np.float32), {}),                               # vmax == vmin
    "vrange": (lambda: field(46, 96, 128, 500.0, 400.0),
               {"vmin": 300.0, "vmax": 1800.5, "azimuths": (45.0,), "sigma_large": 3, "sigma_small": 0.8}),
    "ocean": (lambda: field(47, 80, 72, -3000.0, 400.0), {}),
}


# The golden of a case larger than 64 x 64 keeps every GOLDEN_STRIDE-th row and column, which keeps the fixture small;
# the full images are compared with the oracle, which is pinned to these pixels.
GOLDEN_STRIDE = 2


def golden_stride(name):
    elev, _ = relief_case(name)
    return GOLDEN_STRIDE if elev.size > 64 * 64 else 1


def relief_case(name):
    """(elevation fp32 [H, W], keyword arguments) of one case."""
    build, kw = CASES[name]
    return build(), dict(kw)
