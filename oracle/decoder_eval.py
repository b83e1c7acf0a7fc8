"""ORACLE (test infrastructure, not product): fp32 CPU restatement of one batch of the decoder evaluations.

Reference (xandergos/terrain-diffusion @ 82a0431):
  decoder evaluation loop        terrain_diffusion/evaluation/decoder_consistency.py:108-196
                                 (tiled_decoder_consistency.py:111-201: the same loop at 896 / 512 / 384, then the
                                 centre crop to 512)
  laplacian_decode(pre_padded=True)                  terrain_diffusion/data/laplacian_encoder.py:93-132

Built on the oracle's U-Net (oracle/unet.py), blend window (oracle/tiling.py) and per-plane resize (oracle/postproc.py);
pinned against the reference by tests/golden/make_golden_decoder_eval.py.
"""
from __future__ import annotations

import numpy as np
import torch

from . import postproc as P
from .tiling import accumulate, linear_weight_window, normalise


def readout(residual: np.ndarray, lowfreq_padded: np.ndarray, residual_mean, residual_std, crop=None) -> np.ndarray:
    """One plane: residual [H, W] in normalised units and the pre-padded low-frequency plane [h+2, w+2] -> the terrain
    the drivers hand to the metric (laplacian_decode(pre_padded=True), sign(x) x^2, centre crop), fp32."""
    f32 = np.float32
    hi = (residual.astype(f32) * f32(residual_std) + f32(residual_mean)).astype(f32)
    H, W = hi.shape
    pad = W // (lowfreq_padded.shape[-1] - 2)
    up = P.resize_bilinear(lowfreq_padded.astype(f32), (H + 2 * pad, W + 2 * pad))[pad:-pad, pad:-pad]
    out = (hi + up).astype(f32)
    out = (np.sign(out) * out * out).astype(f32)
    if crop:
        i, j = (H - crop) // 2, (W - crop) // 2
        out = out[i:i + crop, j:j + crop]
    return out


@torch.no_grad()
def decoder_eval_batch(model_fn, t_values, images, lowfreq_padded, cond_img, generator, *, residual_mean,
                       residual_std, sigma_data, tile_size, tile_stride, crop_size=None):
    """model_fn(x[N, 5, T, T], noise_labels[N]) -> [N, 1, T, T]; t_values: the fp32 times of the steps; images
    [B, 1, S, S], lowfreq_padded [B, 1, S/8+2, S/8+2], cond_img [B, 4, S, S]; noise drawn from the CPU `generator` per
    (tile, step).  Returns (generated, real) terrain [B, 1, c, c] fp32."""
    B, C, S, _ = images.shape
    T = tile_size
    weights = linear_weight_window(T)[None, None]
    out, out_w = torch.zeros(images.shape), torch.zeros(images.shape)
    n = (S - T) // tile_stride + 1
    for i in range(n):
        for j in range(n):
            i0, j0 = i * tile_stride, j * tile_stride
            samples = torch.zeros((B, C, T, T))
            tile_cond = cond_img[..., i0:i0 + T, j0:j0 + T]
            for tv in t_values:
                t = torch.tensor(tv, dtype=torch.float32).view(1, 1, 1, 1).expand(B, 1, 1, 1)
                z = torch.randn(samples.shape, generator=generator) * sigma_data
                x_t = torch.cos(t) * samples + torch.sin(t) * z
                pred = -model_fn(torch.cat([x_t / sigma_data, tile_cond], dim=1), t.flatten())
                samples = torch.cos(t) * x_t - torch.sin(t) * sigma_data * pred
            accumulate(out, out_w, samples, weights, i0, j0)
    output = normalise(out, out_w) / sigma_data
    real = images / sigma_data

    def terrain(x):
        return torch.from_numpy(np.stack([readout(x[b, 0].numpy(), lowfreq_padded[b, 0].numpy(), residual_mean,
                                                  residual_std, crop_size) for b in range(B)]))[:, None]
    return terrain(output), terrain(real)
