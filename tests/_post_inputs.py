"""Seeded inputs shared by tests/golden/make_golden_post.py (reference side) and the post-step tests (oracle / CUDA)."""
import numpy as np


def field(seed, h, w, lo=0.0, amp=1.0):
    """Smooth-ish random field: low-frequency sinusoids + white noise (deterministic in numpy, float32)."""
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.zeros((h, w))
    for _ in range(4):
        fy, fx, ph = rng.uniform(0.01, 0.12), rng.uniform(0.01, 0.12), rng.uniform(0, 6.28)
        out += rng.uniform(0.3, 1.0) * np.sin(fy * y + fx * x + ph)
    out += 0.25 * rng.randn(h, w)
    return (lo + amp * out).astype(np.float32)


def laplacian_case(name):
    """(residual [H, W], lowres [h, w]) of the direct laplacian_denoise / laplacian_decode cases."""
    shapes = {"rect": (96, 80, 12, 10), "square": (128, 128, 16, 16), "wide": (64, 136, 8, 17)}
    H, W, h, w = shapes[name]
    seed = sorted(shapes).index(name) + 1
    return field(10 * seed, H, W, 0.0, 3.0), field(10 * seed + 1, h, w, -31.4, 38.6)


class FakeCanvas:
    """canvas[:, a:b, c:d] over world coordinates (negative allowed) -> planes [C+1, b-a, d-c]: values * w and w, like the
    un-normalised (sum x*w, sum w) tensors the pipeline's lazy canvases return."""

    def __init__(self, seed, channels, origin, size, lo, amp):
        self.origin, self.size = origin, size
        h, w = size
        self.wt = (0.5 + np.abs(field(seed + 99, h, w))).astype(np.float32)
        self.val = np.stack([field(seed + c, h, w, lo, amp) for c in range(channels)])

    def planes(self, a, b, c, d):
        oy, ox = self.origin
        assert a >= oy and c >= ox and b <= oy + self.size[0] and d <= ox + self.size[1], "window outside the fake canvas"
        v = self.val[:, a - oy:b - oy, c - ox:d - ox]
        w = self.wt[a - oy:b - oy, c - ox:d - ox]
        return np.concatenate([v * w[None], w[None]], axis=0)


ELEV_WINDOWS = {"neg_square": (-37, 20, 91, 148), "wide": (8, -60, 136, 140), "aligned": (0, 0, 64, 64)}
RESIDUAL_MEAN, RESIDUAL_STD = 0.12, 1.35


def elev_canvases():
    """HR residual canvas (1 value plane + weight) and LR latents canvas (5 value planes + weight), scale 8."""
    resid = FakeCanvas(1000, 1, (-160, -200), (480, 560), 0.0, 0.8)
    lat = FakeCanvas(2000, 5, (-20, -25), (60, 70), 0.2, 0.6)
    return resid, lat


def coarse_canvas():
    """Coarse canvas at 1/256 resolution: 6 value planes (0 = signed-sqrt elevation, 2 = temperature, ...) + weight."""
    c = FakeCanvas(3000, 6, (-12, -12), (30, 32), 0.0, 1.0)
    c.val[0] = field(3100, 30, 32, 5.0, 18.0)        # signed sqrt of metres: the windows ELEV_WINDOWS read are all land
    c.val[2] = field(3200, 30, 32, 12.0, 6.0)        # temperature, deg C
    return c


# A coastal window at scale 2 (coarse stride 64): compute_climate reads coarse rows -11..10 and columns -12..11, and its
# 15 x 15 lapse-rate windows give an 8 x 10 grid of regressions that take every branch of local_baseline_temperature.
COASTAL_WINDOW, COASTAL_SCALE = (-150, -200, 170, 230), 2


def coastal_canvas():
    """Coarse canvas over exactly the rows / columns COASTAL_WINDOW reads: ocean (elevation < 0) everywhere except a
    flat plateau (signed sqrt elevation exactly 1, so var_e < 1) in the top right and steep land in the bottom right
    whose temperature rises with elevation in its top rows and falls fast in its bottom rows.  Windows to the left see
    only ocean (den = 0), windows at the coast see a few land cells (den just below / above 0.02), and the regression
    slopes overshoot both ends of beta_clip."""
    c = FakeCanvas(4000, 6, (-11, -12), (22, 24), 0.0, 1.0)
    e = -(0.5 + np.abs(field(4100, 22, 24)))
    e[0:4, 17:] = 1.0
    e[15:, 17:] = 4.0 + 14.0 * np.abs(field(4200, 7, 7))
    t = field(4300, 22, 24, 12.0, 1.0)
    t[15:17, 17:] = 5.0 + 0.02 * e[15:17, 17:] ** 2 + 0.1 * field(4400, 2, 7)
    t[17:, 17:] = 25.0 - 0.1 * e[17:, 17:] ** 2 + 0.1 * field(4500, 5, 7)
    c.val[0], c.val[2] = e.astype(np.float32), t.astype(np.float32)
    return c


def coastal_coarse_map():
    """(temperature, signed-sqrt elevation) of the normalised coarse map compute_climate builds for COASTAL_WINDOW."""
    i1, j1, i2, j2 = COASTAL_WINDOW
    S = 32 * COASTAL_SCALE
    c = coastal_canvas().planes(i1 // S - 8, -((-i2) // S) + 8, j1 // S - 8, -((-j2) // S) + 8).astype(np.float32)
    cmap = (c[:-1] / c[-1:]).astype(np.float32)
    return cmap[2], cmap[0]


def coastal_elev():
    """Elevation in metres over COASTAL_WINDOW (below sea level in places, so max(elev, 0) clamps)."""
    i1, j1, i2, j2 = COASTAL_WINDOW
    return field(4600, i2 - i1, j2 - j1, 100.0, 400.0)
