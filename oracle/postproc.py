"""TEST ORACLE (not product code): CPU restatement of the reference's elevation read-out -- the "post step" of
SURVEY.md section 8(f) rank 3.  Only tests/, __graft_entry__.smoke() and bench.py's cpu legs may import this.

What it restates (numpy float32, one function per reference function, cited by file:line):
  * WorldPipeline._compute_elev                      terrain_diffusion/inference/world_pipeline.py:1277-1313
  * laplacian_decode / laplacian_encode / laplacian_denoise / resize_extrapolated / pad_linear_extrapolation
                                                     terrain_diffusion/data/laplacian_encoder.py:6-137
  * _elev_to_int16                                   terrain_diffusion/inference/api.py:73-77
  * WorldPipeline._compute_climate                   terrain_diffusion/inference/world_pipeline.py:1314-1365
  * local_baseline_temperature_torch                 terrain_diffusion/inference/postprocessing.py:262-326
    (+ torch's avg_pool2d and grid_sample(bilinear, border, align_corners=False) as they are used there)
and the two third-party pieces those call (not in the reference checkout; torchvision 0.26 / torch 2.11 are installed here,
so the restatement is pinned against the reference run through them -- tests/golden/make_golden_post.py):
  * torchvision.transforms.functional.resize(tensor, size, BILINEAR) -> torch interpolate(mode="bilinear",
    align_corners=False, antialias=True): the separable "anti-aliased" triangle filter of ATen UpSampleKernel.cpp
    (_compute_indices_min_size_weights_aa), last dimension first, for down- AND up-sampling; an int `size` means
    "shorter edge -> size" (torchvision _compute_resized_output_size);
  * torchvision gaussian_blur: reflect padding + the outer product of two normalised 1-D Gaussians on linspace taps.
Parity: pinned (tests/golden/post_golden.npz, max relative deviation ~1e-6: summation order inside torch's conv).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def _aa_weights(in_size: int, out_size: int):
    """ATen _compute_indices_min_size_weights_aa for the triangle filter (interp_size 2), all in float32."""
    scale = F32(in_size) / F32(out_size)
    support = F32(scale) if scale >= 1.0 else F32(1.0)
    invscale = F32(1.0) / scale if scale >= 1.0 else F32(1.0)
    taps = int(np.ceil(support)) * 2 + 1
    xmin = np.zeros(out_size, np.int64)
    xsize = np.zeros(out_size, np.int64)
    wts = np.zeros((out_size, taps), F32)
    for i in range(out_size):
        center = F32(scale * F32(i + 0.5))
        lo = max(int(F32(center - support + F32(0.5))), 0)
        n = min(int(F32(center + support + F32(0.5))), in_size) - lo
        w = np.zeros(taps, F32)
        total = F32(0.0)
        for j in range(n):
            t = F32(F32(j + lo) - center + F32(0.5)) * invscale
            t = -t if t < 0 else t
            w[j] = F32(1.0) - t if t < 1.0 else F32(0.0)
            total = F32(total + w[j])
        if total != 0.0:
            w[:n] = w[:n] / total
        xmin[i], xsize[i], wts[i] = lo, n, w
    return xmin, xsize, wts


def _resize_axis(x: np.ndarray, out_size: int, axis: int) -> np.ndarray:
    x = np.moveaxis(x.astype(F32), axis, -1)
    in_size = x.shape[-1]
    xmin, xsize, wts = _aa_weights(in_size, out_size)
    out = np.zeros(x.shape[:-1] + (out_size,), F32)
    for i in range(out_size):
        acc = x[..., xmin[i]] * wts[i, 0]
        for j in range(1, xsize[i]):
            acc = (acc + x[..., xmin[i] + j] * wts[i, j]).astype(F32)
        out[..., i] = acc
    return np.moveaxis(out, -1, axis)


def resize_bilinear(x: np.ndarray, size) -> np.ndarray:
    """TF.resize(x, size, BILINEAR) on a [H, W] float tensor (antialias=True): W pass, then H pass."""
    h, w = x.shape[-2:]
    if isinstance(size, (tuple, list)):
        new_h, new_w = size
    else:                                   # torchvision: the shorter edge becomes `size`, aspect ratio kept
        short, long = (w, h) if w <= h else (h, w)
        new_short, new_long = int(size), int(int(size) * long / short)
        new_w, new_h = (new_short, new_long) if w <= h else (new_long, new_short)
    if (new_h, new_w) == (h, w):
        return x.astype(F32)
    y = _resize_axis(x, new_w, -1) if new_w != w else x.astype(F32)
    return _resize_axis(y, new_h, -2) if new_h != h else y


def pad_linear_extrapolation(x: np.ndarray) -> np.ndarray:
    """laplacian_encoder.py:6-40: one extrapolated row/column on every side (rows first, then columns of the result)."""
    x = x.astype(F32)
    h, w = x.shape
    top = 2 * x[0:1] - x[1:2] if h > 1 else x[0:1]
    bot = 2 * x[-1:] - x[-2:-1] if h > 1 else x[-1:]
    x = np.concatenate([top, x, bot], axis=0).astype(F32)
    left = 2 * x[:, 0:1] - x[:, 1:2] if w > 1 else x[:, 0:1]
    right = 2 * x[:, -1:] - x[:, -2:-1] if w > 1 else x[:, -1:]
    return np.concatenate([left, x, right], axis=1).astype(F32)


def resize_extrapolated(x: np.ndarray, size) -> np.ndarray:
    """laplacian_encoder.py:42-60."""
    th, tw = size
    h, w = x.shape
    sh, sw = th / h, tw / w
    out = resize_bilinear(pad_linear_extrapolation(x), (int(round(th + 2 * sh)), int(round(tw + 2 * sw))))
    ph, pw = int(round(sh)), int(round(sw))
    return out[ph:ph + th, pw:pw + tw]


def gaussian_kernel1d(kernel_size: int, sigma: float) -> np.ndarray:
    """torchvision _get_gaussian_kernel1d (float32 linspace taps)."""
    half = (kernel_size - 1) * 0.5
    x = np.linspace(-half, half, kernel_size, dtype=F32)
    pdf = np.exp(F32(-0.5) * (x / F32(sigma)) ** 2).astype(F32)
    return (pdf / pdf.sum(dtype=F32)).astype(F32)


def gaussian_blur(x: np.ndarray, kernel_size: int, sigma: float) -> np.ndarray:
    """torchvision gaussian_blur on [H, W]: reflect padding k//2, 2-D kernel = outer(k1d, k1d)."""
    k1 = gaussian_kernel1d(kernel_size, sigma)
    k2 = np.outer(k1, k1).astype(F32)
    p = kernel_size // 2
    xp = np.pad(x.astype(F32), p, mode="reflect")
    h, w = x.shape
    out = np.zeros((h, w), F32)
    for dy in range(kernel_size):
        for dx in range(kernel_size):
            out = (out + k2[dy, dx] * xp[dy:dy + h, dx:dx + w]).astype(F32)
    return out


def kernel_size_for(sigma: float) -> int:
    return int(sigma * 2) // 2 * 2 + 1          # laplacian_encoder.py:75, world_pipeline.py:1286


def laplacian_decode(residual: np.ndarray, lowres: np.ndarray, extrapolate: bool = False) -> np.ndarray:
    """laplacian_encoder.py:95-131 (pre_padded=False)."""
    up = resize_extrapolated(lowres, residual.shape) if extrapolate else resize_bilinear(lowres, residual.shape)
    return (residual.astype(F32) + up).astype(F32)


def laplacian_encode_lowres(x: np.ndarray, downsample_size: int, sigma: float) -> np.ndarray:
    """The `lowres` output of laplacian_encode (laplacian_encoder.py:62-93): resize to an int size, then blur."""
    return gaussian_blur(resize_bilinear(x, downsample_size), kernel_size_for(sigma), sigma)


def laplacian_denoise(residual: np.ndarray, lowres: np.ndarray, sigma: float):
    """laplacian_encoder.py:133-137."""
    decoded = laplacian_decode(residual, lowres, extrapolate=True)
    return residual, laplacian_encode_lowres(decoded, lowres.shape[-1], sigma)


def padded_window(i1: int, j1: int, i2: int, j2: int, scale: int, sigma: float = 5):
    """Integer geometry of _compute_elev (world_pipeline.py:1285-1300): the scale-aligned padded HR window."""
    pad_hr = (kernel_size_for(sigma) // 2 + 1) * scale
    pi1, pj1 = ((i1 - pad_hr) // scale) * scale, ((j1 - pad_hr) // scale) * scale
    pi2, pj2 = -((-(i2 + pad_hr)) // scale) * scale, -((-(j2 + pad_hr)) // scale) * scale
    return pi1, pj1, pi2, pj2


def compute_elev(i1, j1, i2, j2, residual_planes, latents_planes, scale, residual_mean, residual_std,
                 lowfreq_mean=-31.4, lowfreq_std=38.6, sigma=5):
    """world_pipeline.py:1277-1313.  residual_planes(a, b, c, d) -> [2, b-a, d-c] and latents_planes(a, b, c, d) ->
    [C+1, ...] return the un-normalised (sum x*w, sum w) planes of the HR / LR canvases."""
    pi1, pj1, pi2, pj2 = padded_window(i1, j1, i2, j2, scale, sigma)
    r = residual_planes(pi1, pi2, pj1, pj2).astype(F32)
    residual_p = ((r[0] / r[1]) * F32(residual_std) + F32(residual_mean)).astype(F32)
    lat = latents_planes(pi1 // scale, pi2 // scale, pj1 // scale, pj2 // scale).astype(F32)
    lowfreq_p = ((lat[4] / lat[-1]) * F32(lowfreq_std) + F32(lowfreq_mean)).astype(F32)
    residual_p, lowfreq_p = laplacian_denoise(residual_p, lowfreq_p, sigma)
    elev_p = laplacian_decode(residual_p, lowfreq_p)
    oi, oj = i1 - pi1, j1 - pj1
    e = elev_p[oi:oi + (i2 - i1), oj:oj + (j2 - j1)]
    return (np.sign(e) * np.square(e)).astype(F32)


def elev_to_int16(elev: np.ndarray) -> np.ndarray:
    """api.py:73-77.  np.clip keeps a NaN, and numpy's float32 -> int16 cast of NaN is platform-defined: on x86 it goes
    through cvttss2si (NaN -> 0x80000000) and keeps the low 16 bits, so NaN packs as 0.  That x86 result is the one pinned
    here (explicitly, so the oracle gives it on any host) and in tdx_post_combine; +-inf clip to 32767 / -32768."""
    f = np.floor(elev.astype(F32))
    return np.clip(np.where(np.isnan(f), F32(0.0), f), -32768, 32767).astype("<i2")


# ---------------------------------------------------------------------------------------------------- climate read-out
# (groundwork for the device version: restated and pinned, not yet on the GPU path)
def _avg_pool_valid(x: np.ndarray, win: int) -> np.ndarray:
    """F.avg_pool2d(x, win, stride=1, padding=0) on [H, W] (float32 window sum in row-major tap order, / win^2)."""
    h, w = x.shape
    oh, ow = h - win + 1, w - win + 1
    acc = np.zeros((oh, ow), F32)
    for dy in range(win):
        for dx in range(win):
            acc = (acc + x[dy:dy + oh, dx:dx + ow]).astype(F32)
    return (acc / F32(win * win)).astype(F32)


def local_baseline_temperature(T: np.ndarray, e: np.ndarray, win: int, beta_clip=(-0.012, 0.0), fallback_beta=-0.0065,
                               eps=1e-6, fallback_threshold=0.3):
    """inference/postprocessing.py:262-326: land-weighted windowed regression of temperature on elevation."""
    T, e = T.astype(F32), e.astype(F32)
    wmask = (e > 0).astype(F32)
    den = _avg_pool_valid(wmask, win)

    def wavg(x):
        return (_avg_pool_valid((x * wmask).astype(F32), win) / (den + F32(eps))).astype(F32)

    mu_T, mu_e, mu_e2, mu_eT = wavg(T), wavg(e), wavg((e * e).astype(F32)), wavg((e * T).astype(F32))
    var_e = (mu_e2 - mu_e ** 2).astype(F32)
    cov_eT = (mu_eT - mu_e * mu_T).astype(F32)
    beta = (cov_eT / (var_e + F32(eps))).astype(F32)
    invalid = (var_e < 1.0) | (den < fallback_threshold)
    beta = np.where(invalid, F32(fallback_beta), beta).astype(F32)
    beta = np.clip(beta, F32(beta_clip[0]), F32(beta_clip[1])).astype(F32)
    pad = (win - 1) // 2
    T_sea = (T[pad:-pad, pad:-pad] - beta * e[pad:-pad, pad:-pad]).astype(F32)
    return T_sea, beta


def _grid_sample_border(features: np.ndarray, gy: np.ndarray, gx: np.ndarray) -> np.ndarray:
    """F.grid_sample(features[None], grid, mode='bilinear', padding_mode='border', align_corners=False) on [C, H, W]
    with normalised coordinates gy, gx [h, w] (float32 throughout, like ATen's grid sampler)."""
    _, H, W = features.shape
    def unnorm(g, size):
        c = (((g + F32(1.0)) * F32(size)) - F32(1.0)) / F32(2.0)
        return np.clip(c.astype(F32), F32(0.0), F32(size - 1)).astype(F32)
    y, x = unnorm(gy.astype(F32), H), unnorm(gx.astype(F32), W)
    y0, x0 = np.floor(y), np.floor(x)
    wy1, wx1 = (y - y0).astype(F32), (x - x0).astype(F32)
    wy0, wx0 = (F32(1.0) - wy1).astype(F32), (F32(1.0) - wx1).astype(F32)
    y0i, x0i = y0.astype(np.int64), x0.astype(np.int64)
    y1i, x1i = y0i + 1, x0i + 1
    def tap(yi, xi, wgt):
        ok = (yi >= 0) & (yi < H) & (xi >= 0) & (xi < W)
        v = features[:, np.clip(yi, 0, H - 1), np.clip(xi, 0, W - 1)]
        return np.where(ok[None], v * wgt[None], F32(0.0)).astype(F32)
    out = tap(y0i, x0i, (wy0 * wx0).astype(F32))
    out = (out + tap(y0i, x1i, (wy0 * wx1).astype(F32))).astype(F32)
    out = (out + tap(y1i, x0i, (wy1 * wx0).astype(F32))).astype(F32)
    return (out + tap(y1i, x1i, (wy1 * wx1).astype(F32))).astype(F32)


def compute_climate(i1, j1, i2, j2, elev: np.ndarray, coarse_planes, scale: int):
    """world_pipeline.py:1314-1365: [temperature (lapse-rate corrected), coarse ch 3, 4, 5, lapse rate] x [H, W].
    coarse_planes(a, b, c, d) -> [C+1, b-a, d-c] un-normalised planes of the coarse canvas (1/(32*scale) resolution)."""
    S = 32 * scale
    ci1, cj1 = i1 // S, j1 // S
    ci2, cj2 = -((-i2) // S), -((-j2) // S)
    win = 15
    cpad = (win - 1) // 2 + 1
    c = coarse_planes(ci1 - cpad, ci2 + cpad, cj1 - cpad, cj2 + cpad).astype(F32)
    cmap = (c[:-1] / c[-1:]).astype(F32)
    e0 = np.maximum(F32(0.0), cmap[0])
    coarse_elev = (np.sign(cmap[0]) * np.square(e0)).astype(F32)
    t_base, beta = local_baseline_temperature(cmap[2], coarse_elev, win=win, fallback_threshold=0.02)
    central = cmap[:, win // 2:-(win // 2), win // 2:-(win // 2)]
    Hs, Ws = t_base.shape
    ii = np.arange(i1, i2, dtype=np.int64)[:, None] + np.zeros((1, j2 - j1), np.int64)
    jj = np.arange(j1, j2, dtype=np.int64)[None, :] + np.zeros((i2 - i1, 1), np.int64)
    u = (((ii.astype(F32) + F32(0.5)) / F32(S)) - F32(ci1) + F32(0.5)).astype(F32)
    v = (((jj.astype(F32) + F32(0.5)) / F32(S)) - F32(cj1) + F32(0.5)).astype(F32)
    gy = (((u + F32(0.5)) * F32(2.0)) / F32(Hs) - F32(1.0)).astype(F32)
    gx = (((v + F32(0.5)) * F32(2.0)) / F32(Ws) - F32(1.0)).astype(F32)
    feats = np.concatenate([t_base[None], beta[None], central], axis=0).astype(F32)
    up = _grid_sample_border(feats, gy, gx)
    t_real = (up[0] + up[1] * np.maximum(elev.astype(F32), F32(0.0))).astype(F32)
    return np.stack([t_real, up[2 + 3], up[2 + 4], up[2 + 5], up[1]]).astype(F32)
