"""ORACLE (test infrastructure, not product): fp32 CPU restatement of the evaluation drivers' terrain decode.

Reference (xandergos/terrain-diffusion @ 82a0431):
  _decode_latents_to_terrain    terrain_diffusion/evaluation/base_consistency.py:34-72 (the same function in
                                base_diffusion.py and the infinite_consistency*.py drivers)
  _normalize_uint8_three_channel                                  base_consistency.py:25-32

Built on the oracle's consistency sampler (oracle/tiling.py) and the per-plane Laplacian read-out (oracle/postproc.py);
pinned against the reference by tests/golden/make_golden_eval_terrain.py.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import postproc as P
from .tiling import sample_decoder_consistency_tiled

LOWFREQ_MEAN, LOWFREQ_STD = -31.4, 38.6


def readout(residual: np.ndarray, lowfreq: np.ndarray, residual_mean, residual_std, denoise: bool = True,
            signed_square: bool = False) -> np.ndarray:
    """One image: residual [H, W] and lowfreq [h, w] in normalised units -> terrain [H, W] (fp32)."""
    f32 = np.float32
    hi = (residual.astype(f32) * f32(residual_std) + f32(residual_mean)).astype(f32)
    lo = (lowfreq.astype(f32) * f32(LOWFREQ_STD) + f32(LOWFREQ_MEAN)).astype(f32)
    if denoise:
        hi, lo = P.laplacian_denoise(hi, lo, sigma=5)
    out = P.laplacian_decode(hi, lo, extrapolate=True)
    return (np.sign(out) * out * out).astype(f32) if signed_square else out


@torch.no_grad()
def decode_latents_to_terrain(model_fn, sigma0, sigma_data, samples, latents_mean, latents_std, residual_mean,
                              residual_std, noise, inter_t=(), denoise: bool = True) -> torch.Tensor:
    """model_fn(x[N,5,T,T], noise_labels[N]) -> [N,1,T,T]; samples [B, 5, h, w]; noise: the unit draw [B, 1, 8h, 8w].
    Returns [B, 1, 8h, 8w] fp32."""
    latents, lowfreq = samples[:, :4], samples[:, 4:5]
    latents = latents / latents_std + latents_mean
    H, W = lowfreq.shape[-2] * 8, lowfreq.shape[-1] * 8
    cond = F.interpolate(latents, size=(H, W), mode="nearest")
    residual = sample_decoder_consistency_tiled(model_fn, sigma_data, sigma0, cond, noise, H, H,
                                                intermediate_t=tuple(inter_t))
    out = [readout(residual[b, 0].numpy(), lowfreq[b, 0].numpy(), residual_mean, residual_std, denoise)
           for b in range(samples.shape[0])]
    return torch.from_numpy(np.stack(out))[:, None]


def normalize_uint8_three_channel(images: torch.Tensor) -> torch.Tensor:
    image_min = torch.amin(images, dim=(1, 2, 3), keepdim=True)
    image_max = torch.amax(images, dim=(1, 2, 3), keepdim=True)
    image_range = torch.maximum(image_max - image_min, torch.tensor(255.0))
    image_mid = (image_min + image_max) / 2
    normalized = torch.clamp(((images - image_mid) / image_range + 0.5) * 255, 0, 255)
    return normalized.repeat(1, 3, 1, 1).to(torch.uint8)
