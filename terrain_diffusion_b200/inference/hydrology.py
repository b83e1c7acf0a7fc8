"""River routing on the device: drop-ins for `d8_flow`, `flow_accumulation` and `plot_flow_indicator` of
terrain_diffusion.inference.postprocessing (postprocessing.py:6-85).  `plot_flow_indicator` is the `flow` input the
relief map compares with `flow_threshold` to draw rivers.  `fill_depressions_priority_flood` and `smooth_river_bumps`
(postprocessing.py:87-260, csrc/tdx_depress.cu) prepare an elevation for routing: filled pits drain instead of ending
rivers in sinks.  They accept +-inf, which behaves as in the reference.

The reference runs D8 routing as a numpy stencil and the accumulation as a Python loop over every land pixel in
descending elevation order.  Here each is one pass of csrc/tdx_hydro.cu.  Every edge the accumulation follows is
strictly downhill, so its result is the order-independent integer sum A = 1 + (the A of every pixel draining in), which the
device computes exactly under any thread schedule: the outputs are bit-identical to the reference's.

Conventions (as inference/relief.py): a numpy array or CPU tensor is computed on the current CUDA device and numpy is
returned, with the reference's dtypes; a CUDA tensor returns torch tensors on its own device, computed on its current
stream.  `z` must be a 2-D float array of at most 2^24 pixels without +inf; it is computed in fp32 (a float64 `z` is
rounded to fp32 first).  -inf is ocean, as in the reference: its slopes are all overwritten by the ocean rules.  +inf
is rejected because a +inf pixel next to another has the NaN slope inf - inf, and the reference's argmax then depends
on where that NaN sits.  Argument errors raise ValueError before any device work, except the +inf check of a CUDA
tensor, which reads one 4-byte flag back after the launches.
"""
from __future__ import annotations

import ctypes as C
import math
import operator

import numpy as np
import torch

from .. import _lib as L

MAX_PIXELS = 1 << 24         # fp32 counts are exact integers up to here
_FLAG_INF, _FLAG_RANGE, _FLAG_NOT_DOWNHILL = 1, 2, 4   # tdx.h TDX_FLOW_*
FILL_BATCH = 32              # tdx.h TDX_FILL_BATCH: flag words of the fill's pass batches


def _shape(x) -> tuple:
    return tuple(x.shape) if hasattr(x, "shape") else np.shape(x)


def _elevation(z, fn: str, name: str = "z", finite: bool = True):
    """(fp32 z, on_device): a contiguous CUDA tensor when z is one, else a host numpy array, after every check that
    needs no device.  finite=False accepts +inf (-inf is always accepted: it is ocean)."""
    if isinstance(z, torch.Tensor):
        floating = z.is_floating_point()
    else:
        z = np.asarray(z)
        floating = np.issubdtype(z.dtype, np.floating)
    shape = _shape(z)
    if len(shape) != 2 or shape[0] < 1 or shape[1] < 1:
        raise ValueError(f"{fn}: {name} must be 2-D (H, W) with H, W >= 1, got shape {shape}")
    if shape[0] * shape[1] > MAX_PIXELS:
        raise ValueError(f"{fn}: at most 2^24 pixels (fp32 counts are exact up to there), got {shape}")
    if not floating:
        raise ValueError(f"{fn}: {name} must be a float array, got {z.dtype}")
    if isinstance(z, torch.Tensor) and z.is_cuda:
        return z.detach().to(torch.float32).contiguous(), True
    host = z.detach().cpu().numpy() if isinstance(z, torch.Tensor) else z
    with np.errstate(over="ignore"):
        host = np.ascontiguousarray(host, dtype=np.float32)
    if finite and np.isposinf(host).any():
        raise ValueError(f"{fn}: z has +inf elevations (in fp32); their slopes are NaN and the result would depend on "
                         "the visiting order")
    return host, False


def _on_device(host: np.ndarray) -> torch.Tensor:
    if not torch.cuda.is_available():
        raise L.TdxError("river routing runs on a CUDA device and none is available (there is no CPU path)")
    return torch.from_numpy(host).cuda()


def _check_flags(flags: torch.Tensor, fn: str) -> None:
    f = int(flags)
    if f & _FLAG_INF:
        raise ValueError(f"{fn}: z has +inf elevations (in fp32); their slopes are NaN and the result would depend on "
                         "the visiting order")
    if f & _FLAG_RANGE:
        raise ValueError(f"{fn}: a receiver index rr / cc lies outside the image")
    if f & _FLAG_NOT_DOWNHILL:
        raise ValueError(f"{fn}: a followed receiver (valid, non-sink source into a valid target) is not strictly "
                         "lower than its source, so the accumulation would depend on the visiting order")


def d8_flow(z, tol=1e-3):
    """Steepest-descent (D8) receivers: (rr, cc, is_sink, kmax), int64 / int64 / bool / int64 [H, W], bit-identical
    to the reference.  Neighbours N, S, W, E, NW, NE, SW, SE are read edge-clamped; a slope below tol (compared in
    fp32, as NumPy 2 does) does not count; ocean (NaN or <= 0) neighbours are preferred outlets."""
    zz, on_device = _elevation(z, "d8_flow")
    with np.errstate(over="ignore"):
        tol32 = float(np.float32(tol))
    zd = zz if on_device else _on_device(zz)
    h, w = zd.shape
    kw = dict(device=zd.device)
    kmax = torch.empty((h, w), dtype=torch.int8, **kw)
    sink = torch.empty((h, w), dtype=torch.uint8, **kw)
    rr = torch.empty((h, w), dtype=torch.int64, **kw)
    cc = torch.empty((h, w), dtype=torch.int64, **kw)
    flags = torch.empty(1, dtype=torch.int32, **kw)
    L.call(L.lib().tdx_flow_d8, zd.device, zd.data_ptr(), h, w, tol32, kmax.data_ptr(), sink.data_ptr(), rr.data_ptr(),
           cc.data_ptr(), None, None, flags.data_ptr())
    if on_device:
        _check_flags(flags, "d8_flow")
        return rr, cc, sink.view(torch.bool), kmax.long()
    return rr.cpu().numpy(), cc.cpu().numpy(), sink.cpu().numpy().view(bool), kmax.cpu().numpy().astype(np.int64)


def _receiver_array(x, name: str, shape: tuple, flag: bool):
    """rr / cc (integer) or is_sink (bool or integer, flag=True) after the host checks: its shape is z's."""
    if _shape(x) != shape:
        raise ValueError(f"flow_accumulation: {name} has shape {_shape(x)}, z has {shape}")
    if isinstance(x, torch.Tensor):
        integer = not (x.is_floating_point() or x.is_complex() or x.dtype == torch.bool)
        ok = integer or (flag and x.dtype == torch.bool)
    else:
        x = np.asarray(x)
        ok = np.issubdtype(x.dtype, np.integer) or (flag and x.dtype == np.bool_)
    if not ok:
        kind = "a bool or integer" if flag else "an integer"
        raise ValueError(f"flow_accumulation: {name} must be {kind} array, got {x.dtype}")
    return x


def _to_device(x, device, dtype) -> torch.Tensor:
    if dtype == torch.uint8:                                   # is_sink: any non-zero value is a sink
        x = (x != 0) if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x) != 0)
    elif not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.int64))
    return x.detach().to(device=device, dtype=dtype).contiguous()


def flow_accumulation(z, rr, cc, is_sink):
    """Upstream cell count of every pixel, fp32 [H, W]: 1 + the counts of the pixels that drain into it for valid
    (not NaN, > 0) pixels, 0 elsewhere.  A pixel drains into (rr, cc) when it is valid, not a sink and (rr, cc) is
    valid.  The output follows z: numpy for host z, a tensor on z's device for CUDA z; rr / cc / is_sink may come from
    anywhere and are moved there.

    The one deviation from the reference: every index must lie in the image and every followed edge must be strictly
    downhill in fp32, else ValueError (one 4-byte flag read back after the check runs on the device).  The reference
    silently returns a result that depends on its visiting order for such receivers.  Receivers from either
    project's `d8_flow` always pass."""
    zz, on_device = _elevation(z, "flow_accumulation")
    shape = tuple(zz.shape)
    rr, cc = _receiver_array(rr, "rr", shape, False), _receiver_array(cc, "cc", shape, False)
    is_sink = _receiver_array(is_sink, "is_sink", shape, True)
    zd = zz if on_device else _on_device(zz)
    h, w = shape
    rd, cd = _to_device(rr, zd.device, torch.int64), _to_device(cc, zd.device, torch.int64)
    sd = _to_device(is_sink, zd.device, torch.uint8)
    recv = torch.empty((h, w), dtype=torch.int32, device=zd.device)
    indeg = torch.empty((h, w), dtype=torch.int32, device=zd.device)
    flags = torch.empty(1, dtype=torch.int32, device=zd.device)
    L.call(L.lib().tdx_flow_link, zd.device, zd.data_ptr(), rd.data_ptr(), cd.data_ptr(), sd.data_ptr(), h, w,
           recv.data_ptr(), indeg.data_ptr(), flags.data_ptr())
    _check_flags(flags, "flow_accumulation")
    a = _accumulate(zd, recv, indeg)
    return a if on_device else a.cpu().numpy()


def _accumulate(zd, recv, indeg) -> torch.Tensor:
    state = torch.empty(zd.numel(), dtype=torch.int64, device=zd.device)
    a = torch.empty(zd.shape, dtype=torch.float32, device=zd.device)
    L.call(L.lib().tdx_flow_accumulate, zd.device, zd.data_ptr(), zd.numel(), recv.data_ptr(), indeg.data_ptr(),
           state.data_ptr(), a.data_ptr())
    return a


def plot_flow_indicator(z, max_pool_kernel=1):
    """log1p of the upstream cell counts of d8_flow(z) (default tol), zero on invalid pixels, after a non-overlapping
    max_pool_kernel x max_pool_kernel max-pool that drops the remainder rows and columns (no pool for a kernel <= 1):
    fp32 [H // k, W // k], empty when k exceeds H or W, as in the reference.  Three launches on one stream; a CUDA
    input reads back only the 4-byte +inf flag."""
    zz, on_device = _elevation(z, "plot_flow_indicator")
    try:
        k = operator.index(max_pool_kernel)
    except TypeError:
        raise ValueError(f"plot_flow_indicator: max_pool_kernel must be an integer, got {max_pool_kernel!r}") from None
    k = max(k, 1)
    zd = zz if on_device else _on_device(zz)
    h, w = zd.shape
    recv = torch.empty((h, w), dtype=torch.int32, device=zd.device)
    indeg = torch.empty((h, w), dtype=torch.int32, device=zd.device)
    flags = torch.empty(1, dtype=torch.int32, device=zd.device)
    L.call(L.lib().tdx_flow_d8, zd.device, zd.data_ptr(), h, w, float(np.float32(1e-3)), None, None, None, None,
           recv.data_ptr(), indeg.data_ptr(), flags.data_ptr())
    a = _accumulate(zd, recv, indeg)
    out = torch.empty((h // k, w // k), dtype=torch.float32, device=zd.device)
    L.call(L.lib().tdx_flow_indicator, zd.device, a.data_ptr(), h, w, k, out.data_ptr())
    if on_device:
        _check_flags(flags, "plot_flow_indicator")
        return out
    return out.cpu().numpy()


def _is_fp32(x) -> bool:
    return x.dtype == (torch.float32 if isinstance(x, torch.Tensor) else np.float32)


def _nodata32(nodata) -> float:
    """The fp32 value `h == nodata` matches, as NumPy 2 compares a float32 array with it: a Python number is rounded to
    fp32; a NumPy scalar compares in its own precision, so one that fp32 cannot hold matches nothing (NaN)."""
    if nodata is None:
        return float("nan")
    with np.errstate(over="ignore"):
        v = np.float32(nodata)
    if isinstance(nodata, np.generic) and not np.isnan(v) and v != nodata:
        return float("nan")
    return float(v)


def _fill(hd: torch.Tensor, eps32: float, connectivity: int, nodata32: float):
    """(filled fp32 tensor on hd's device, relaxation passes) of a contiguous fp32 CUDA tensor."""
    h, w = hd.shape
    out = torch.empty_like(hd)
    kind = torch.empty((h, w), dtype=torch.uint8, device=hd.device)
    flags = torch.empty(FILL_BATCH, dtype=torch.int32, device=hd.device)
    passes = C.c_int32(0)
    L.call(L.lib().tdx_fill_depressions, hd.device, hd.data_ptr(), h, w, eps32, connectivity, nodata32, out.data_ptr(),
           kind.data_ptr(), flags.data_ptr(), C.byref(passes))
    return out, passes.value


def fill_depressions_priority_flood(height, epsilon=1e-3, max_raise=None, connectivity=8, in_place=False,
                                    nodata=None):
    """Priority-Flood depression fill with an epsilon gradient across flats, bit-identical to the reference for
    max_raise=None: fp32 [H, W].  Invalid pixels (NaN, <= 0 or == nodata, compared in fp32) keep their height, and so
    do the seeds: valid border pixels and valid pixels with an invalid neighbour.  Every other pixel becomes
    h if h > m else max(h, m + epsilon) (one fp32 add), m being the lowest filled value among its valid neighbours
    (connectivity 4: N, S, W, E; any other value: all 8).  +inf is land, -inf is invalid.

    This is the fixed point the device relaxes to from +inf (csrc/tdx_depress.cu); it reads one flag back per batch
    of passes, so the call synchronises the stream.  in_place=True writes the result into a float32 `height` (array
    or tensor) and returns it, as the reference does for a float32 ndarray; other dtypes are left untouched.
    max_raise other than None raises NotImplementedError, epsilon < 0 or not finite ValueError, both before any
    device work."""
    fn = "fill_depressions_priority_flood"
    if max_raise is not None:
        raise NotImplementedError(
            f"{fn}: max_raise={max_raise!r} is not supported, only None: a capped fill pushes cells below the current "
            "flood level and its basin minima depend on which neighbour arrives first, so its result follows the "
            "heap's visiting order and has no order-free (parallel) form")
    try:
        eps = float(epsilon)
    except (TypeError, ValueError):
        raise ValueError(f"{fn}: epsilon must be a number, got {epsilon!r}") from None
    if not (math.isfinite(eps) and eps >= 0):
        raise ValueError(f"{fn}: epsilon must be finite and >= 0, got {epsilon!r}: with a negative epsilon the "
                         "flood's pops are no longer in order and its result depends on the visiting order")
    hh, on_device = _elevation(height, fn, "height", finite=False)
    with np.errstate(over="ignore"):
        eps32 = float(np.float32(eps))                      # NumPy 2 adds a Python float to a float32 in fp32
    nodata32 = _nodata32(nodata)
    hd = hh if on_device else _on_device(hh)
    out, _ = _fill(hd, eps32, 4 if connectivity == 4 else 8, nodata32)
    if in_place and _is_fp32(height):
        if isinstance(height, torch.Tensor):
            height.detach().copy_(out)
            return height if on_device else height.detach().numpy()
        np.copyto(height, out.cpu().numpy())
        return height
    return out if on_device else out.cpu().numpy()


def smooth_river_bumps(height, slope_thresh=50, smooth_strength=0.3, iterations=3):
    """`iterations` steps of h += smooth_strength * exp(-(slope / slope_thresh)^2) * laplace(h) on the pixels that
    are not NaN in `height`, fp32 [H, W] (H, W >= 2), NaN pixels kept NaN.  slope is |np.gradient| (central
    differences inside, one-sided at the edges) and laplace the 4-neighbour Laplacian over the non-NaN neighbours,
    which wrap around the edges as np.roll does.  Every fp32 operation is rounded separately in numpy's order and exp
    is evaluated in fp64 and rounded once, so a pixel can differ from numpy's SIMD fp32 exp by that function's error
    (about 2 ulp of the weight).  One launch per iteration."""
    fn = "smooth_river_bumps"
    try:
        iters = operator.index(iterations)
    except TypeError:
        raise ValueError(f"{fn}: iterations must be an integer, got {iterations!r}") from None
    if iters >= 2 ** 31:
        raise ValueError(f"{fn}: iterations must be below 2^31, got {iters}")
    hh, on_device = _elevation(height, fn, "height", finite=False)
    if min(hh.shape) < 2:
        raise ValueError(f"{fn}: height needs at least 2 rows and 2 columns (np.gradient), got {tuple(hh.shape)}")
    with np.errstate(over="ignore"):
        thresh32, strength32 = float(np.float32(slope_thresh)), float(np.float32(smooth_strength))
    hd = hh if on_device else _on_device(hh)
    out = torch.empty_like(hd)
    scratch = torch.empty_like(hd) if iters > 1 else None
    L.call(L.lib().tdx_smooth_river_bumps, hd.device, hd.data_ptr(), hd.shape[0], hd.shape[1], thresh32, strength32,
           max(iters, 0), out.data_ptr(), None if scratch is None else scratch.data_ptr())
    return out if on_device else out.cpu().numpy()
