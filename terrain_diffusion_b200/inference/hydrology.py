"""River routing on the device: drop-ins for `d8_flow`, `flow_accumulation` and `plot_flow_indicator` of
terrain_diffusion.inference.postprocessing (postprocessing.py:6-85).  `plot_flow_indicator` is the `flow` input the
relief map compares with `flow_threshold` to draw rivers.

The reference runs D8 routing as a numpy stencil and the accumulation as a Python loop over every land pixel in
descending elevation order.  Here each is one pass of csrc/tdx_hydro.cu.  Every edge the accumulation follows is
strictly downhill, so its result is the order-independent integer sum A = 1 + (the A of every pixel draining in), which the
device computes exactly under any thread schedule: the outputs are bit-identical to the reference's.

Conventions (as inference/relief.py): a numpy array or CPU tensor is computed on the current CUDA device and numpy is
returned, with the reference's dtypes; a CUDA tensor returns torch tensors on its own device, computed on its current
stream.  `z` must be a 2-D float array of at most 2^24 pixels without +-inf; it is computed in fp32 (a float64 `z` is
rounded to fp32 first).  Argument errors raise ValueError before any device work, except the +-inf check of a CUDA
tensor, which reads one 4-byte flag back after the launches.
"""
from __future__ import annotations

import operator

import numpy as np
import torch

from .. import _lib as L

MAX_PIXELS = 1 << 24         # fp32 counts are exact integers up to here
_FLAG_INF, _FLAG_RANGE, _FLAG_NOT_DOWNHILL = 1, 2, 4   # tdx.h TDX_FLOW_*


def _shape(x) -> tuple:
    return tuple(x.shape) if hasattr(x, "shape") else np.shape(x)


def _elevation(z, fn: str):
    """(fp32 z, on_device): a contiguous CUDA tensor when z is one, else a host numpy array, after every check that
    needs no device."""
    if isinstance(z, torch.Tensor):
        floating = z.is_floating_point()
    else:
        z = np.asarray(z)
        floating = np.issubdtype(z.dtype, np.floating)
    shape = _shape(z)
    if len(shape) != 2 or shape[0] < 1 or shape[1] < 1:
        raise ValueError(f"{fn}: z must be 2-D (H, W) with H, W >= 1, got shape {shape}")
    if shape[0] * shape[1] > MAX_PIXELS:
        raise ValueError(f"{fn}: at most 2^24 pixels (fp32 counts are exact up to there), got {shape}")
    if not floating:
        raise ValueError(f"{fn}: z must be a float array, got {z.dtype}")
    if isinstance(z, torch.Tensor) and z.is_cuda:
        return z.detach().to(torch.float32).contiguous(), True
    host = z.detach().cpu().numpy() if isinstance(z, torch.Tensor) else z
    with np.errstate(over="ignore"):
        host = np.ascontiguousarray(host, dtype=np.float32)
    if np.isinf(host).any():
        raise ValueError(f"{fn}: z has +-inf elevations (in fp32); their slopes are NaN and the result would depend on "
                         "the visiting order")
    return host, False


def _on_device(host: np.ndarray) -> torch.Tensor:
    if not torch.cuda.is_available():
        raise L.TdxError("river routing runs on a CUDA device and none is available (there is no CPU path)")
    return torch.from_numpy(host).cuda()


def _check_flags(flags: torch.Tensor, fn: str) -> None:
    f = int(flags)
    if f & _FLAG_INF:
        raise ValueError(f"{fn}: z has +-inf elevations (in fp32); their slopes are NaN and the result would depend on "
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
    input reads back only the 4-byte +-inf flag."""
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
