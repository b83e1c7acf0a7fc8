"""Seeded elevation windows of the river-routing cases, shared by tests/golden/make_golden_hydrology.py (reference side)
and the hydrology tests (oracle / CUDA)."""
import numpy as np

from tests._post_inputs import field


def _mixed():
    e = field(61, 96, 128, 150.0, 400.0)                     # land and ocean
    rng = np.random.RandomState(62)
    e.flat[rng.choice(e.size, 60, replace=False)] = np.nan
    e[30:34, 40:70] = np.nan
    return e


def _plateau():
    # elevations on a 25 m grid: exact-tie plateaus (flat sinks), equal slopes in several directions (the k-order
    # tie-break), exact 0 and -0.0 ocean
    e = np.round(field(63, 64, 80, 40.0, 60.0) / np.float32(25.0)) * np.float32(25.0)
    e[50:54, 10:20] = -0.0
    return e.astype(np.float32)


def _edge_ocean():
    # all land except ocean pixels on the border rows and columns, which the border pixels read both directly and
    # through the edge-clamped neighbours of the padded stencil
    e = field(64, 40, 48, 900.0, 120.0)
    e[0, 10:13] = -5.0
    e[17:21, -1] = np.nan
    e[-1, 0] = 0.0
    e[-1, 30] = -1.0
    e[5, 0] = np.nan
    return e


def _two():
    return np.array([[2.0, 1.0], [1.0, 1.0]], np.float32)   # equal N/W slopes into ties; the flat corner is a sink


def _tol_between():
    # slopes are exact multiples of 0.125; tol lies between fp32(0.125) and the next fp32 value, so a slope of exactly
    # 0.125 survives an fp32 comparison and would not survive a float64 one
    rng = np.random.RandomState(65)
    steps = np.cumsum(rng.randint(0, 3, size=(24, 32)), axis=1) + np.cumsum(rng.randint(0, 2, size=(24, 1)), axis=0)
    return (np.float32(40.0) + np.float32(0.125) * steps.astype(np.float32)).astype(np.float32)


def _big():
    e = smooth_field(256, seed=66)                           # long rivers
    e[100:103, :] = np.nan
    return e


def _neg_inf():
    # -inf ocean next to land, NaN, 0.0 and -0.0, on the border rows and columns, in all four corners, as one-pixel
    # lakes and as a block whose inner pixels see only -inf
    e = field(84, 40, 48, 400.0, 150.0)
    e[5:12, 6:14] = -np.inf
    e[8, 14] = np.nan                                         # NaN beside -inf
    e[12, 6:10] = 0.0
    e[12, 10:14] = -0.0
    e[0, 20:25] = -np.inf
    e[-1, 30:33] = -np.inf
    e[15:19, 0] = -np.inf
    e[22:24, -1] = -np.inf
    e[0, 0] = e[0, -1] = e[-1, 0] = e[-1, -1] = -np.inf
    e[25, 25] = e[30, 12] = e[33, 40] = -np.inf
    return e


def _neg_inf_seams():
    # -inf on the rows and columns where the device's 32 x 8 tiles meet (rows 7 | 8, 15 | 16, columns 31 | 32, 63 | 64)
    e = field(85, 20, 70, 300.0, 120.0)
    e[7, 20:40] = -np.inf
    e[16, 28:36] = -np.inf
    e[2:18, 32] = -np.inf
    e[8:12, 63] = -np.inf
    e[15, 60:66] = np.nan
    return e


CASES = {
    # name: (elevation builder, d8 tol, max-pool kernels of the indicator)
    "mixed": (_mixed, 1e-3, (0, 1, 3)),
    "plateau": (_plateau, 1e-3, (1, 2)),
    "edge_ocean": (_edge_ocean, 1e-3, (1, 8)),
    "all_nan": (lambda: np.full((8, 8), np.nan, np.float32), 1e-3, (1, 8)),
    "all_ocean": (lambda: np.minimum(field(67, 12, 16, -300.0, 100.0), np.float32(0.0)), 1e-3, (1, 2)),
    "row": (lambda: field(68, 1, 37, 100.0, 80.0), 1e-3, (1, 2)),          # k = 2 > H: an empty (0, 18) result
    "col": (lambda: field(69, 29, 1, 60.0, 70.0), 1e-3, (1, 3)),
    "two": (_two, 1e-3, (1, 3)),
    "tol_large": (lambda: field(70, 48, 40, 500.0, 300.0), 5.0, (1,)),
    "tol_between": (_tol_between, 0.125 + 1e-9, (1,)),
    "big": (_big, 1e-3, (1, 3, 8)),
    "neg_inf": (_neg_inf, 1e-3, (1, 3)),
    "neg_inf_seams": (_neg_inf_seams, 1e-3, (1, 2)),
    "neg_inf_all": (lambda: np.full((5, 6), -np.inf, np.float32), 1e-3, (1, 2)),
}


def _neg_inf_pits():
    # smooth terrain with dug pits and -inf ocean: the fill keeps the ocean at -inf and routing must accept it
    e = field(86, 56, 72, 250.0, 200.0)
    rng = np.random.RandomState(87)
    for _ in range(15):
        y, x = rng.randint(3, 53), rng.randint(3, 69)
        e[y - 2:y + 2, x - 2:x + 3] -= np.float32(rng.uniform(20, 200))
    e[e < 5] = -np.inf
    e[40:56, 0:12] = -np.inf
    e.flat[rng.choice(e.size, 20, replace=False)] = np.nan
    return e


# routed after the reference's fill_depressions_priority_flood (default arguments): name -> (elevation builder, pools).
# The golden stores the filled window as `<name>.filled` next to the routing outputs.
FILLED_CASES = {
    "neg_inf_filled": (_neg_inf_pits, (1, 2)),
}


def hydrology_case(name):
    """(elevation fp32 [H, W], tol, pool kernels) of one case."""
    build, tol, pools = CASES[name]
    return build(), tol, pools


def smooth_field(n, seed=0, ocean_fraction=0.125):
    """Seeded smooth n x n terrain in metres with about `ocean_fraction` of it NaN ocean, the kind of window the relief
    map draws rivers on."""
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:n, 0:n].astype(np.float64) / n
    e = np.zeros((n, n))
    for _ in range(6):
        e += rng.uniform(300, 900) * np.sin(rng.uniform(2, 20) * y + rng.uniform(2, 20) * x + rng.uniform(0, 6.28))
    e += 5.0 * rng.randn(n, n)
    e = e - np.quantile(e, ocean_fraction) + 1.0
    e[e <= 0] = np.nan
    return e.astype(np.float32)


def serpentine(n):
    """Adversarial n x n ramp (n even): every pixel drains into one outlet through a single boustrophedon flow path of
    n * n / 2 + n / 2 - 1 cells.  Rows 0, 2, ... are channels falling 1 m per pixel, alternately east and west; each
    odd row is a ridge, except for one turning pixel at the channel's end, entered with a 0.25 m drop (so the diagonal
    into it is never steeper than the channel) and left with a 4 m drop (so the diagonal past the next channel's first
    pixel is never steeper).  Ridge pixels drain into the channel next to them.  Returns (z, path as flat indices)."""
    assert n % 2 == 0 and n >= 4
    path, drops = [], []
    for r in range(0, n, 2):
        cols = range(n) if (r // 2) % 2 == 0 else range(n - 1, -1, -1)
        for i, c in enumerate(cols):
            path.append(r * n + c)
            drops.append(4.0 if (i == 0 and r > 0) else 1.0)
        if r + 2 < n:
            path.append((r + 1) * n + cols[-1])
            drops.append(0.25)
    below = np.cumsum(np.asarray(drops[:0:-1]))[::-1]      # below[i] = drops[i + 1] + ... : the fall after cell i
    z_path = np.float64(1.0) + np.concatenate([below, [0.0]])
    z = np.full(n * n, z_path[0] + 100.0)
    z[np.asarray(path)] = z_path
    assert z_path[0] + 100.0 < 2 ** 24 / 4                  # quarter-metre steps stay exact in fp32
    return z.reshape(n, n).astype(np.float32), np.asarray(path)
