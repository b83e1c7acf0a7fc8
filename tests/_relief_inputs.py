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


def _inf_case():
    e = field(48, 32, 40, 400.0, 300.0)
    e[4, 5] = np.inf
    e[26, 33] = -np.inf
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
    # branches the cases above do not reach
    "inf": (_inf_case, {"sigma_large": 1.5, "sigma_small": 0.5}),        # +-inf: fallback range, NaN around +inf
    "relief2": (lambda: field(49, 24, 32, 300.0, 900.0), {"relief": 2.0}),  # gain < 0 on dark slopes, clipped to 0
    "vmin_only": (lambda: field(50, 24, 32, 300.0, 600.0), {"vmin": 500.0}),  # one bound alone: the data's range
    "vmax_only": (lambda: field(51, 24, 32, 300.0, 600.0), {"vmax": 700.0}),
    "vmin_above": (lambda: field(52, 24, 32, 400.0, 300.0), {"vmin": 5000.0, "vmax": 9000.0}),  # land is black
    "abyss": (lambda: field(54, 24, 32, -8000.0, 3000.0), {}),                # below -10000 m: the depth clip
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


def bench_field(n: int) -> np.ndarray:
    """The elevation tools/bench_relief.py renders at n x n (a copy of its seeded builder): a smooth field with land
    and ocean."""
    rng = np.random.RandomState(n)
    y, x = np.mgrid[0:n, 0:n].astype(np.float64) / n
    e = np.zeros((n, n))
    for _ in range(6):
        e += rng.uniform(300, 900) * np.sin(rng.uniform(2, 20) * y + rng.uniform(2, 20) * x + rng.uniform(0, 6.28))
    return (e + 200 + 30 * rng.randn(n, n)).astype(np.float32)
