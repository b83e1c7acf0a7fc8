"""Elevation read-out on the device (SURVEY.md section 8(f) rank 3).

Mirrors, function for function, what the reference runs on the CPU for every `WorldPipeline.get()`:
`data/laplacian_encoder.py` (pad_linear_extrapolation :6-40, resize_extrapolated :42-60, laplacian_encode :62-93,
laplacian_decode :95-131, laplacian_denoise :133-137), `WorldPipeline._compute_elev` (inference/world_pipeline.py:
1277-1313) and `_elev_to_int16` (inference/api.py:73-77).  The torchvision calls inside them (`TF.resize` = torch's
anti-aliased separable bilinear filter, `TF.gaussian_blur`) are the fp32 kernels of csrc/tdx_post.cu; tensors are
CUDA fp32 `[H, W]` and never leave the GPU.  There is no CPU path: CPU tensors raise.
"""
from __future__ import annotations

import ctypes as C

import functools

import numpy as np
import torch

from .. import _lib as L

LOWFREQ_MEAN, LOWFREQ_STD = -31.4, 38.6          # world_pipeline.py:1280-1281


def _on_arg_device(fn):
    """Run `fn` with the CUDA device of its first device-carrying argument (tensor or canvas) current: libtdx launches
    on the current device and on its current stream (L.current_stream_ptr())."""
    @functools.wraps(fn)
    def wrapper(*a, **k):
        for v in list(a) + list(k.values()):
            dev = getattr(v, "device", None)
            if isinstance(dev, torch.device) and dev.type == "cuda":
                with torch.cuda.device(dev):
                    return fn(*a, **k)
        return fn(*a, **k)
    return wrapper


def _chk(x: torch.Tensor, name: str) -> torch.Tensor:
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 2):
        raise L.TdxError(f"{name}: expected a CUDA float32 [H, W] tensor (the GPU read-out has no CPU path), got "
                         f"{getattr(x, 'device', None)} {getattr(x, 'dtype', None)} {tuple(getattr(x, 'shape', ()))}")
    return x.contiguous()


def _p(t: torch.Tensor):
    return C.c_void_p(t.data_ptr())


def _resized_output_size(h: int, w: int, size) -> tuple[int, int]:
    """torchvision's rule: a (h, w) pair is taken as is; an int is the new length of the SHORTER edge."""
    if isinstance(size, (tuple, list, torch.Size)):
        return int(size[0]), int(size[1])
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = int(size), int(int(size) * long / short)
    new_w, new_h = (new_short, new_long) if w <= h else (new_long, new_short)
    return new_h, new_w


@_on_arg_device
def resize_bilinear(x: torch.Tensor, size) -> torch.Tensor:
    """TF.resize(x, size, interpolation=BILINEAR) for an fp32 tensor (antialias on): width pass, then height pass."""
    x = _chk(x, "resize_bilinear")
    h, w = x.shape
    new_h, new_w = _resized_output_size(h, w, size)
    s = L.current_stream_ptr()
    if new_w != w:
        y = torch.empty((h, new_w), dtype=torch.float32, device=x.device)
        L.check(L.lib().tdx_resize_aa_axis(_p(x), h, w, _p(y), new_w, 1, s))
        x, w = y, new_w
    if new_h != h:
        y = torch.empty((new_h, w), dtype=torch.float32, device=x.device)
        L.check(L.lib().tdx_resize_aa_axis(_p(x), h, w, _p(y), new_h, 0, s))
        x = y
    return x


@_on_arg_device
def pad_linear_extrapolation(x: torch.Tensor) -> torch.Tensor:
    x = _chk(x, "pad_linear_extrapolation")
    h, w = x.shape
    out = torch.empty((h + 2, w + 2), dtype=torch.float32, device=x.device)
    L.check(L.lib().tdx_post_pad_extrapolate(_p(x), h, w, _p(out), L.current_stream_ptr()))
    return out


def resize_extrapolated(x: torch.Tensor, size) -> torch.Tensor:
    """laplacian_encoder.py:42-60 for a (h, w) target: pad by linear extrapolation, resize, crop the pad away."""
    th, tw = int(size[0]), int(size[1])
    h, w = x.shape
    sh, sw = th / h, tw / w
    out = resize_bilinear(pad_linear_extrapolation(x), (int(round(th + 2 * sh)), int(round(tw + 2 * sw))))
    ph, pw = int(round(sh)), int(round(sw))
    return out[ph:ph + th, pw:pw + tw]


@_on_arg_device
def gaussian_blur(x: torch.Tensor, kernel_size: int, sigma: float) -> torch.Tensor:
    x = _chk(x, "gaussian_blur")
    h, w = x.shape
    out = torch.empty_like(x)
    L.check(L.lib().tdx_gaussian_blur(_p(x), h, w, _p(out), int(kernel_size), float(sigma), L.current_stream_ptr()))
    return out


@_on_arg_device
def _combine(a: torch.Tensor, b: torch.Tensor, signed_square: bool = False, int16: bool = False):
    """f(a + b) over two equally shaped (possibly strided-row) views."""
    assert a.shape == b.shape and a.stride(1) == 1 and b.stride(1) == 1
    h, w = a.shape
    out = torch.empty((h, w), dtype=torch.float32, device=a.device)
    out16 = torch.empty((h, w), dtype=torch.int16, device=a.device) if int16 else None
    L.check(L.lib().tdx_post_combine(_p(a), a.stride(0), _p(b), b.stride(0), _p(out),
                                     _p(out16) if int16 else None, h, w, int(signed_square), L.current_stream_ptr()))
    return (out, out16) if int16 else out


def laplacian_decode(residual: torch.Tensor, lowres: torch.Tensor, extrapolate: bool = False) -> torch.Tensor:
    """residual + upsampled lowres (laplacian_encoder.py:95-131, pre_padded=False)."""
    residual = _chk(residual, "laplacian_decode")
    up = resize_extrapolated(lowres, residual.shape) if extrapolate else resize_bilinear(lowres, tuple(residual.shape))
    return _combine(residual, up)


def kernel_size_for(sigma: float) -> int:
    return int(sigma * 2) // 2 * 2 + 1


def laplacian_encode_lowres(x: torch.Tensor, downsample_size: int, sigma: float) -> torch.Tensor:
    """The `lowres` result of laplacian_encode (laplacian_encoder.py:62-93): resize to an int size, then blur."""
    return gaussian_blur(resize_bilinear(x, downsample_size), kernel_size_for(sigma), sigma)


def laplacian_denoise(residual: torch.Tensor, lowres: torch.Tensor, sigma: float):
    decoded = laplacian_decode(residual, lowres, extrapolate=True)
    return residual, laplacian_encode_lowres(decoded, lowres.shape[-1], sigma)


def padded_window(i1: int, j1: int, i2: int, j2: int, scale: int, sigma: float = 5):
    """The scale-aligned padded window _compute_elev reads (world_pipeline.py:1285-1300); floor / ceil division."""
    pad_hr = (kernel_size_for(sigma) // 2 + 1) * scale
    pi1, pj1 = ((i1 - pad_hr) // scale) * scale, ((j1 - pad_hr) // scale) * scale
    pi2, pj2 = -((-(i2 + pad_hr)) // scale) * scale, -((-(j2 + pad_hr)) // scale) * scale
    return pi1, pj1, pi2, pj2


@_on_arg_device
def compute_elev(residual_canvas, latents_canvas, i1: int, j1: int, i2: int, j2: int, scale: int, residual_mean: float,
                 residual_std: float, sigma: float = 5, as_int16: bool = False):
    """Elevation in metres over pixel rows [i1, i2) x columns [j1, j2) (world_pipeline.py:1277-1313).

    The canvases are indexed like the reference's lazy tensors -- `canvas[:, a:b, c:d]` returns the un-normalised
    (sum x*w ..., sum w) planes as a CUDA tensor -- `residual_canvas` at pixel resolution (2 planes), `latents_canvas`
    at 1/scale resolution (channel 4 = low-frequency elevation, last plane = weight).  Returns fp32 [i2-i1, j2-j1]
    (and, with as_int16, also the clip(floor(.)) int16 tensor of api.py:73-77)."""
    if i2 <= i1 or j2 <= j1:
        raise ValueError("Expected i2>i1 and j2>j1")
    pi1, pj1, pi2, pj2 = padded_window(i1, j1, i2, j2, scale, sigma)
    r = residual_canvas[:, pi1:pi2, pj1:pj2]
    lat = latents_canvas[:, pi1 // scale:pi2 // scale, pj1 // scale:pj2 // scale]
    if not (r.is_cuda and lat.is_cuda):
        raise L.TdxError("compute_elev: the canvases must return CUDA tensors (no CPU path)")
    r, lat = r.float().contiguous(), lat.float().contiguous()
    hp, wp = r.shape[-2:]
    hl, wl = lat.shape[-2:]
    s = L.current_stream_ptr()
    residual_p = torch.empty((hp, wp), dtype=torch.float32, device=r.device)
    lowfreq_p = torch.empty((hl, wl), dtype=torch.float32, device=r.device)
    L.check(L.lib().tdx_post_normalize(_p(r[0]), _p(r[1]), wp, _p(residual_p), hp, wp, float(residual_std),
                                       float(residual_mean), s))
    L.check(L.lib().tdx_post_normalize(_p(lat[4]), _p(lat[-1]), wl, _p(lowfreq_p), hl, wl, LOWFREQ_STD, LOWFREQ_MEAN, s))
    residual_p, lowfreq_p = laplacian_denoise(residual_p, lowfreq_p, sigma)
    up = resize_bilinear(lowfreq_p, (hp, wp))
    oi, oj = i1 - pi1, j1 - pj1
    h, w = i2 - i1, j2 - j1
    return _combine(residual_p[oi:oi + h, oj:oj + w], up[oi:oi + h, oj:oj + w], signed_square=True, int16=as_int16)


def terrain_window(i1: int, j1: int, i2: int, j2: int, scale: int):
    """Checks the arguments of a terrain request (api.py:68-69, 193-194) and returns the native window `_get_terrain`
    reads and the crop origin in its upsampled version (api.py:114-153): (ni1, nj1, ni2, nj2, oi, oj).  The window is
    padded by one native pixel on every side for scale > 1; Python floor / ceil division, so negative coordinates work.

    Raises ValueError for a non-integer coordinate or scale, scale < 1, an empty window (i2 <= i1 or j2 <= j1) or more
    than 65535 output rows.  The reference raises for an empty window only at scale 1; above it, it returns wrongly
    sliced tensors."""
    for name, v in (("i1", i1), ("j1", j1), ("i2", i2), ("j2", j2), ("scale", scale)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError(f"{name} must be an int, got {v!r}")
    i1, j1, i2, j2, scale = int(i1), int(j1), int(i2), int(j2), int(scale)
    if scale < 1:
        raise ValueError("scale must be >= 1")
    if i2 <= i1 or j2 <= j1:
        raise ValueError("Expected i2>i1 and j2>j1")
    if i2 - i1 > 65535:
        raise ValueError(f"at most 65535 rows per request, got {i2 - i1}")
    if scale == 1:
        return i1, j1, i2, j2, 0, 0
    ni1, nj1 = i1 // scale, j1 // scale
    ni2, nj2 = -(-i2 // scale), -(-j2 // scale)
    return ni1 - 1, nj1 - 1, ni2 + 1, nj2 + 1, scale + (i1 - ni1 * scale), scale + (j1 - nj1 * scale)


@_on_arg_device
def upsample_crop(elev: torch.Tensor, climate: torch.Tensor | None, scale: int, oi: int, oj: int, H: int, W: int,
                  payload: bool = False) -> torch.Tensor:
    """The terrain API's upsample + crop (api.py:139-164, torch's CPU F.interpolate(scale_factor=scale, mode='bilinear',
    align_corners=False) bit for bit) of the native window `elev` [h, w] (and `climate` [5, h, w]), output pixels
    [oi, oi+H) x [oj, oj+W) of the upsampled window only; scale == 1 is the plain crop.  Returns one CUDA tensor: fp32
    [6, H, W] (elevation, then the 5 climate planes) or [1, H, W] without climate; with `payload`, the wire body of
    api.py:80-100 as uint8 [2HW (+ 16HW with climate)]."""
    elev = _chk(elev, "upsample_crop(elev)")
    h, w = elev.shape
    if climate is not None:
        if not (isinstance(climate, torch.Tensor) and climate.is_cuda and climate.dtype == torch.float32
                and tuple(climate.shape) == (5, h, w) and climate.device == elev.device):
            raise L.TdxError(f"upsample_crop: climate must be a CUDA float32 [5, {h}, {w}] tensor on {elev.device}")
        climate = climate.contiguous()
    s = L.current_stream_ptr()
    clim_p = _p(climate) if climate is not None else None
    if payload:
        out = torch.empty((H * W * (18 if climate is not None else 2),), dtype=torch.uint8, device=elev.device)
        L.check(L.lib().tdx_terrain_upsample(_p(elev), clim_p, h, w, scale, oi, oj, H, W, None, None, _p(out), s))
        return out
    out = torch.empty((6 if climate is not None else 1, H, W), dtype=torch.float32, device=elev.device)
    L.check(L.lib().tdx_terrain_upsample(_p(elev), clim_p, h, w, scale, oi, oj, H, W, _p(out[0]),
                                         _p(out[1]) if climate is not None else None, None, s))
    return out


@_on_arg_device
def to_host(t: torch.Tensor) -> torch.Tensor:
    """One device -> host copy into pinned memory (torch's caching host allocator), on the current stream, waited for."""
    staging = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    staging.copy_(t, non_blocking=True)
    torch.cuda.current_stream(t.device).synchronize()
    return staging


@_on_arg_device
def compute_climate(coarse_canvas, i1: int, j1: int, i2: int, j2: int, elev: torch.Tensor, scale: int) -> torch.Tensor:
    """Climate over pixel rows [i1, i2) x columns [j1, j2) (WorldPipeline._compute_climate, world_pipeline.py:1314-1365):
    fp32 CUDA [5, H, W] = {temperature with the local lapse-rate correction, coarse channels 3, 4, 5, lapse rate}.

    `coarse_canvas[:, a:b, c:d]` returns the un-normalised planes of the coarse canvas (one cell = 32*scale pixels; channel
    0 = signed-sqrt elevation, 2 = temperature, last = weight); `elev` is compute_elev's result for the same window."""
    elev = _chk(elev, "compute_climate(elev)")
    if tuple(elev.shape) != (i2 - i1, j2 - j1):
        raise ValueError(f"elev is {tuple(elev.shape)}, the window is {(i2 - i1, j2 - j1)}")
    S = 32 * scale
    ci1, cj1 = i1 // S, j1 // S
    ci2, cj2 = -((-i2) // S), -((-j2) // S)
    win = 15                                           # coarse_window_size (world_pipeline.py:1324)
    cpad = (win - 1) // 2 + 1
    c = coarse_canvas[:, ci1 - cpad:ci2 + cpad, cj1 - cpad:cj2 + cpad]
    if not c.is_cuda:
        raise L.TdxError("compute_climate: the coarse canvas must return CUDA tensors (no CPU path)")
    c = c.float().contiguous()
    nch, hc, wc = c.shape[0] - 1, c.shape[1], c.shape[2]
    s = L.current_stream_ptr()
    cmap = torch.empty((nch, hc, wc), dtype=torch.float32, device=c.device)
    for k in range(nch):                               # coarse_map = coarse_init[:-1] / coarse_init[-1:]
        L.check(L.lib().tdx_post_normalize(_p(c[k]), _p(c[-1]), wc, _p(cmap[k]), hc, wc, 1.0, 0.0, s))
    hs, ws = hc - win + 1, wc - win + 1
    t_sea = torch.empty((hs, ws), dtype=torch.float32, device=c.device)
    beta = torch.empty((hs, ws), dtype=torch.float32, device=c.device)
    # local_baseline_temperature_torch(coarse_map[2], coarse_elev_denorm, win=15, fallback_threshold=0.02), defaults of
    # inference/postprocessing.py:262-270 otherwise
    L.check(L.lib().tdx_lapse_rate(_p(cmap[2]), _p(cmap[0]), hc, wc, win, -0.012, 0.0, -0.0065, 1e-6, 0.02, _p(t_sea),
                                   _p(beta), s))
    out = torch.empty((5, i2 - i1, j2 - j1), dtype=torch.float32, device=c.device)
    L.check(L.lib().tdx_climate_sample(_p(t_sea), _p(beta), _p(cmap), nch, hc, wc, win // 2, _p(elev), i1, j1, i2 - i1,
                                       j2 - j1, S, ci1, cj1, _p(out), s))
    return out
