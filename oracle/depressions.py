"""CPU restatement of the reference's depression fill and river-bed smoothing (inference/postprocessing.py:87-260) in
vectorised numpy.

`fill` is the fixed point the reference's Priority-Flood computes for max_raise=None and epsilon >= 0: invalid pixels
(NaN, <= 0, == nodata) and seeds (valid border pixels, valid pixels with an invalid neighbour) keep h, and every
other pixel is G(h, m) = h if h > m else max(h, fl32(m + fl32(eps))), m being the minimum over its valid neighbours.
It is found by Jacobi passes from +inf.  `fill_ordered` computes the same fixed point in increasing order with a heap
(one settle per pixel), for inputs whose longest raised chain would take the Jacobi passes too long.  `smooth` follows
numpy's operation order with exp evaluated in fp64 and rounded once.  Pinned against the reference's own functions
by tests/golden/depressions_golden.npz; the device kernels are checked against this module."""
from __future__ import annotations

import heapq

import numpy as np

OFFSETS8 = ((-1, 0), (1, 0), (0, -1), (0, 1), (-1, -1), (-1, 1), (1, -1), (1, 1))


def offsets(connectivity):
    return OFFSETS8[:4] if connectivity == 4 else OFFSETS8


def classify(height, connectivity=8, nodata=None):
    """(fp32 h, invalid, seed) of the flood."""
    h = np.array(height, dtype=np.float32)
    with np.errstate(invalid="ignore"):
        invalid = np.isnan(h) | (h <= 0)
        if nodata is not None:
            invalid |= h == nodata                         # NumPy 2: a Python number compares in fp32
    H, W = h.shape
    pad = np.pad(invalid, 1, constant_values=False)         # outside the image is not ocean
    coast = np.zeros_like(invalid)
    for dy, dx in offsets(connectivity):
        coast |= pad[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
    border = np.zeros_like(invalid)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    seed = ~invalid & (border | coast)
    return h, invalid, seed


def _g(h, m, eps):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.where(h > m, h, np.maximum(h, m + eps))


def fill(height, epsilon=1e-3, connectivity=8, nodata=None):
    """(filled fp32 [H, W], Jacobi passes run, the last one changing nothing)."""
    h, invalid, seed = classify(height, connectivity, nodata)
    free = ~invalid & ~seed
    eps = np.float32(epsilon)
    out = np.where(free, np.float32(np.inf), h)
    H, W = h.shape
    passes = 0
    while True:
        passes += 1
        pad = np.pad(np.where(invalid, np.float32(np.inf), out), 1, constant_values=np.inf)
        m = np.full((H, W), np.inf, np.float32)
        for dy, dx in offsets(connectivity):
            m = np.minimum(m, pad[1 + dy:1 + dy + H, 1 + dx:1 + dx + W])
        new = np.where(free, _g(h, m, eps), out)
        if np.array_equal(new, out, equal_nan=True):
            return out, passes
        out = new


def fill_ordered(height, epsilon=1e-3, connectivity=8, nodata=None):
    """The same fixed point, settled in increasing order from the seeds (a label-setting shortest path: G is
    monotone and never below m).  Python loop; about a second per 2^18 pixels."""
    h, invalid, seed = classify(height, connectivity, nodata)
    H, W = h.shape
    eps = np.float32(epsilon)
    out = np.where(invalid | seed, h, np.float32(np.inf)).ravel()
    hf, inv = h.ravel(), invalid.ravel()
    done = inv | seed.ravel()
    heap = [(float(out[i]), int(i)) for i in np.flatnonzero(seed.ravel())]
    heapq.heapify(heap)
    nbrs = offsets(connectivity)
    while heap:
        v, i = heapq.heappop(heap)
        if v != out[i]:                                      # superseded by a lower push
            continue
        done[i] = True
        m = np.float32(v)
        raised = m + eps                                     # fp32
        r, c = divmod(i, W)
        for dy, dx in nbrs:
            y, x = r + dy, c + dx
            if 0 <= y < H and 0 <= x < W:
                j = y * W + x
                if not done[j]:
                    hj = hf[j]
                    g = hj if hj > m else max(hj, raised)
                    if g < out[j]:
                        out[j] = g
                        heapq.heappush(heap, (float(g), j))
    return out.reshape(H, W)


def smooth(height, slope_thresh=50, smooth_strength=0.3, iterations=3):
    """smooth_river_bumps in fp32, numpy's operation order, exp in fp64 rounded once."""
    h = np.array(height, dtype=np.float32)
    nan = np.isnan(h)
    t, s = np.float32(slope_thresh), np.float32(smooth_strength)
    zero = np.float32(0)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for _ in range(iterations):
            hs = np.where(nan, zero, h)
            gy, gx = np.gradient(hs)                      # fp32: (f[i+1] - f[i-1]) / 2 inside, one-sided at the edges
            slope = np.sqrt(gx * gx + gy * gy)
            ok = [np.roll(~nan, shift, axis) for shift, axis in ((1, 0), (-1, 0), (1, 1), (-1, 1))]   # up dn lf rt
            nb = [np.where(k, np.roll(hs, shift, axis), zero)
                  for k, (shift, axis) in zip(ok, ((1, 0), (-1, 0), (1, 1), (-1, 1)))]
            total = ((nb[0] + nb[1]) + nb[2]) + nb[3]
            count = ((ok[0].astype(np.float32) + ok[1]) + ok[2]) + ok[3]
            lap = np.where(nan, zero, total - count * hs)
            q = slope / t
            w = np.exp((-(q * q)).astype(np.float64)).astype(np.float32)
            w[nan] = 0
            h = h + (s * w) * lap
            h[nan] = np.nan
    return h
