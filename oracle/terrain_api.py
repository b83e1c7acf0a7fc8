"""TEST ORACLE (not product code): CPU restatement of the HTTP API's terrain read-out, terrain_diffusion/inference/api.py
`_get_terrain` (:103-166) and `_binary_response` (:80-100), and of the torch CPU bilinear kernels `_get_terrain` calls.
Only tests/ and tools may import this.  Parity: pinned bit for bit (tests/golden/terrain_api_golden.npz).
"""
from __future__ import annotations

import numpy as np

from oracle.postproc import elev_to_int16

F32 = np.float32


# ------------------------------------------------------------------------------------------- terrain API read-out
# api.py:103-166 (_get_terrain) upsamples the padded native window with torch's CPU F.interpolate(scale_factor=scale,
# mode='bilinear', align_corners=False).  ATen has two CPU kernels for it and picks by the size of the whole upsampled
# window (UpSampleKernel.cpp, _use_vectorized_kernel_cond_2d): out_h + out_w <= 128 takes the kernel with per-pixel
# 2-D weights, larger windows the separable generic kernel.  The x86 builds contract a*b + c into fma, and the two
# kernels contract differently.  Both are pinned against torch 2.11 (AVX512 dispatch) by terrain_api_golden.npz.
def fma32(a, b, c) -> np.ndarray:
    """fp32 fused multiply-add, correctly rounded: a*b is exact in fp64, and the one case where rounding the fp64 sum to
    fp32 would round twice (the fp64 sum lies exactly halfway between two floats but the exact sum does not) is
    resolved with the exact error of the fp64 addition."""
    a, b, c = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)                     # p + c == s + e exactly (TwoSum)
        r = s.astype(F32)
        d = s - r.astype(np.float64)
        nb = np.nextafter(r, np.where(d > 0, F32(np.inf), F32(-np.inf)).astype(F32))
        tie = np.isfinite(s) & np.isfinite(r) & (d != 0) & ((nb.astype(np.float64) - s) == d) & (e != 0)
        return np.where(tie & (np.sign(e) == np.sign(d)), nb, r).astype(F32)


def upsample_taps(n: int, scale: int, dst: np.ndarray):
    """Source indices and weights of output indices `dst` along one axis of length n (area_pixel_compute_source_index
    + guard_index_and_lambda, ATen UpSample.h): (i0, i1, l0, l1)."""
    r = F32(1.0 / scale)
    src = np.maximum(fma32(r, (dst.astype(F32) + F32(0.5)).astype(F32), F32(-0.5)), F32(0.0))
    i0 = np.minimum(np.floor(src).astype(np.int64), n - 1)
    i1 = i0 + (i0 < n - 1)
    l1 = np.clip((src - i0.astype(F32)).astype(F32), F32(0.0), F32(1.0)).astype(F32)
    return i0, i1, (F32(1.0) - l1).astype(F32), l1


def upsample_crop(x: np.ndarray, scale: int, oi: int, oj: int, H: int, W: int) -> np.ndarray:
    """F.interpolate(x[None], scale_factor=scale, mode='bilinear', align_corners=False)[0][..., oi:oi+H, oj:oj+W] for
    x [..., h, w] fp32, bit for bit with torch's CPU result, evaluated at the kept pixels only.  scale == 1 is the crop."""
    x = np.asarray(x, F32)
    h, w = x.shape[-2:]
    if scale == 1:
        return x[..., oi:oi + H, oj:oj + W].copy()
    hi0, hi1, hl0, hl1 = upsample_taps(h, scale, np.arange(oi, oi + H))
    wi0, wi1, wl0, wl1 = upsample_taps(w, scale, np.arange(oj, oj + W))
    x00, x01 = x[..., hi0[:, None], wi0[None, :]], x[..., hi0[:, None], wi1[None, :]]
    x10, x11 = x[..., hi1[:, None], wi0[None, :]], x[..., hi1[:, None], wi1[None, :]]
    hl0, hl1, wl0, wl1 = hl0[:, None], hl1[:, None], wl0[None, :], wl1[None, :]
    with np.errstate(invalid="ignore", over="ignore"):
        if (h + w) * scale <= 128:                       # cpu_upsample_linear_channels_last: 2-D weights, a sum of four
            w00, w01 = (hl0 * wl0).astype(F32), (hl0 * wl1).astype(F32)
            w10, w11 = (hl1 * wl0).astype(F32), (hl1 * wl1).astype(F32)
            o = fma32(w00, x00, (w01 * x01).astype(F32))
            return fma32(w11, x11, fma32(w10, x10, o))
        # upsample_generic_Nd_kernel_impl / Interpolate<2>: rows of the width pass, then the height pass
        t0 = fma32(wl0, x00, (wl1 * x01).astype(F32))
        t1 = fma32(wl0, x10, (wl1 * x11).astype(F32))
        return fma32(hl0, t0, (hl1 * t1).astype(F32))


def terrain_window(i1: int, j1: int, i2: int, j2: int, scale: int):
    """api.py:114-153: the native window _get_terrain reads and the crop origin in the upsampled window:
    (ni1, nj1, ni2, nj2, oi, oj).  Python floor / ceil division, so negative coordinates work."""
    if scale == 1:
        return i1, j1, i2, j2, 0, 0
    ni1, nj1 = i1 // scale, j1 // scale
    ni2, nj2 = -(-i2 // scale), -(-j2 // scale)
    return ni1 - 1, nj1 - 1, ni2 + 1, nj2 + 1, scale + (i1 - ni1 * scale), scale + (j1 - nj1 * scale)


def terrain_payload(elev: np.ndarray, climate) -> bytes:
    """api.py:80-100 _binary_response's body: int16-LE elevation, then climate[:4] as interleaved fp32-LE [H][W][4]."""
    body = elev_to_int16(elev).tobytes()
    if climate is not None and climate.shape[0] >= 4:
        body += np.ascontiguousarray(np.transpose(np.asarray(climate[:4], "<f4"), (1, 2, 0))).tobytes()
    return body
