"""CPU restatement of the reference's river routing (inference/postprocessing.py:6-85) in vectorised numpy.

`d8` evaluates the eight neighbours one direction at a time with a running first-maximum instead of a stacked argmax;
`accumulate` sums upstream counts level by level over the receiver forest (Kahn's order: a pixel pushes its count
once every pixel draining into it has pushed), in int64.  That equals the reference's descending-elevation loop
exactly whenever every followed edge is strictly downhill, which d8 guarantees for tol > 0.  Pinned against the
reference's own functions by tests/golden/hydrology_golden.npz; the device kernels are checked against this module."""
from __future__ import annotations

import numpy as np

# neighbour k = N, S, W, E, NW, NE, SW, SE as (dy, dx)
OFFSETS = ((-1, 0), (1, 0), (0, -1), (0, 1), (-1, -1), (-1, 1), (1, -1), (1, 1))
DIAGONAL = np.float32(np.sqrt(2.0))


def ocean(z: np.ndarray) -> np.ndarray:
    """NaN or <= 0 (-0.0 included): a sink centre, a preferred outlet as a neighbour, never counted."""
    return np.isnan(z) | (z <= 0)


def d8(z, tol=1e-3):
    """(rr, cc, is_sink, kmax) of d8_flow for fp32 z: int64, int64, bool, int64 [H, W]."""
    z = np.asarray(z, dtype=np.float32)
    h, w = z.shape
    t = np.float32(tol)                                     # NumPy 2 compares the fp32 slopes with fp32(tol)
    ys, xs = np.arange(h)[:, None], np.arange(w)[None, :]
    centre_ocean = ocean(z)
    best = np.full((h, w), -np.inf, np.float32)
    kmax = np.zeros((h, w), np.int64)
    any_ocean = np.zeros((h, w), bool)
    any_slope = np.zeros((h, w), bool)
    for k, (dy, dx) in enumerate(OFFSETS):
        nb = z[np.clip(ys + dy, 0, h - 1), np.clip(xs + dx, 0, w - 1)]
        nb_ocean = ocean(nb)
        with np.errstate(invalid="ignore"):
            slope = (z - nb) / (np.float32(1.0) if k < 4 else DIAGONAL)
            slope = np.where(slope < t, np.float32(-np.inf), slope)
        land = ~centre_ocean & ~nb_ocean
        any_ocean |= nb_ocean
        any_slope |= land & np.isfinite(slope)
        prefer = np.where(centre_ocean, -np.inf, np.where(nb_ocean, np.inf, slope)).astype(np.float32)
        better = prefer > best                              # strict: the first maximum keeps its k
        best = np.where(better, prefer, best)
        kmax[better] = k
    is_sink = centre_ocean | (~any_ocean & ~any_slope)
    dys = np.array([o[0] for o in OFFSETS])
    dxs = np.array([o[1] for o in OFFSETS])
    rr = np.clip(ys + dys[kmax], 0, h - 1)
    cc = np.clip(xs + dxs[kmax], 0, w - 1)
    return rr, cc, is_sink, kmax


def receivers(z, rr, cc, is_sink) -> np.ndarray:
    """Flat receiver of every pixel whose count flow_accumulation moves (valid, not a sink, valid target), else -1."""
    z = np.asarray(z, dtype=np.float32)
    valid = ~ocean(z).ravel()
    target = (np.asarray(rr) * z.shape[1] + np.asarray(cc)).ravel()
    push = valid & ~np.asarray(is_sink, bool).ravel() & valid[target]
    return np.where(push, target, -1)


def accumulate(z, rr, cc, is_sink) -> np.ndarray:
    """flow_accumulation: fp32 [H, W] upstream cell counts (1 + the counts draining in) on valid pixels, 0 elsewhere.
    Requires every followed edge to be strictly downhill (asserted)."""
    z = np.asarray(z, dtype=np.float32)
    recv = receivers(z, rr, cc, is_sink)
    src = np.flatnonzero(recv >= 0)
    flat = z.ravel()
    assert np.all(flat[recv[src]] < flat[src]), "a followed edge is not strictly downhill"
    a = (~ocean(flat)).astype(np.int64)
    waiting = np.bincount(recv[src], minlength=flat.size)   # children that have not pushed yet
    front = src[waiting[src] == 0]
    while front.size:
        dst = recv[front]
        np.add.at(a, dst, a[front])
        np.add.at(waiting, dst, -1)
        dst = np.unique(dst)
        done = dst[waiting[dst] == 0]
        front = done[recv[done] >= 0]
    return a.reshape(z.shape).astype(np.float32)


def indicator(a, z, max_pool_kernel=1) -> np.ndarray:
    """log1p of the counts with invalid pixels zeroed, after a non-overlapping k x k max-pool (k > 1) that drops the
    remainder rows and columns."""
    a = np.where(ocean(np.asarray(z, np.float32)), np.float32(0), np.asarray(a, np.float32))
    k = int(max_pool_kernel)
    if k > 1:
        hh, ww = a.shape[0] // k, a.shape[1] // k
        a = a[:hh * k, :ww * k].reshape(hh, k, ww, k).max(axis=(1, 3))
    return np.log1p(a)


def flow_indicator(z, max_pool_kernel=1) -> np.ndarray:
    rr, cc, is_sink, _ = d8(z)
    return indicator(accumulate(z, rr, cc, is_sink), z, max_pool_kernel)
