"""ORACLE (test infrastructure, not product): fp32 CPU restatement of the reference's two-model guided samplers.

Reference (xandergos/terrain-diffusion @ 82a0431):
  _scale_score                                  terrain_diffusion/training/evaluation/sample_diffusion_decoder.py:7-40
  sample_decoder_diffusion_tiled (guided)       .../sample_diffusion_decoder.py:44-125 (guide :112-117, scaling :119)
  _process_cond_img                             terrain_diffusion/training/evaluation/sample_diffusion_base.py:11-48
  sample_base_diffusion                         .../sample_diffusion_base.py:51-168 (guide :105-110, :155-160)

Pinned against the reference by tests/golden/make_golden_guided.py.  The guided decoder sampler is restated with the
per-tile scheduler reset of oracle.tiling.sample_decoder_diffusion_tiled (the shipped function fails on a second tile,
SURVEY.md section 0 item 7); the goldens use one tile, where both agree.
"""
from __future__ import annotations

import numpy as np
import torch

from .tiling import accumulate, linear_weight_window, normalise, tile_starts
from .unet import mp_concat


def scale_score(model_output, sample, sigma, sigma_data: float, alpha: float = 1.0):
    if alpha == 1.0:
        return model_output
    v_t = -sigma_data * model_output
    sigma = torch.as_tensor(sigma, dtype=sample.dtype)
    while sigma.ndim < sample.ndim:
        sigma = sigma.view(*sigma.shape, *([1] * (sample.ndim - sigma.ndim)))
    sdata = torch.as_tensor(sigma_data, dtype=sample.dtype)
    t = torch.atan(sigma / sdata)
    cos_t, sin_t = torch.cos(t), torch.sin(t)
    x0_pred = sample * cos_t - v_t * sin_t
    noise_pred = sample * sin_t + v_t * cos_t
    x0_alpha = sample + alpha * (x0_pred - sample)
    v_t_alpha = noise_pred * cos_t - x0_alpha * sin_t
    return v_t_alpha / -sdata


def guided(model_fn, guide_fn, guidance_scale, *args):
    """sample_diffusion_decoder.py:112-117: the guide is skipped when absent or at scale 1."""
    if guide_fn is None or guidance_scale == 1.0:
        return model_fn(*args)
    mo_m = model_fn(*args)
    mo_g = guide_fn(*args)
    return mo_g + guidance_scale * (mo_m - mo_g)


@torch.no_grad()
def sample_decoder_diffusion_tiled(model_fn, make_scheduler, cond_img, noise, tile_size=None, tile_stride=None,
                                   num_steps=20, guide_fn=None, guidance_scale=1.0, score_scaling=1.0):
    """model_fn / guide_fn(x[N,5,h,w], noise_labels[N]) -> [N,1,h,w]."""
    b, c, h, w = noise.shape
    tile_size = tile_size or min(h, w)
    tile_stride = tile_stride or tile_size
    weights = linear_weight_window(tile_size, noise.dtype)[None, None]
    out = torch.zeros_like(noise)
    out_w = torch.zeros_like(noise)
    for i0 in tile_starts(h, tile_size, tile_stride):
        for j0 in tile_starts(w, tile_size, tile_stride):
            sch = make_scheduler()
            sch.set_timesteps(num_steps)
            samples = noise[..., i0:i0 + tile_size, j0:j0 + tile_size]
            tile_cond = cond_img[..., i0:i0 + tile_size, j0:j0 + tile_size]
            for t, sigma in zip(sch.timesteps, sch.sigmas):
                scaled = sch.precondition_inputs(samples, sigma)
                cnoise = sch.trigflow_precondition_noise(sigma.view(-1).expand(b))
                mo = guided(model_fn, guide_fn, guidance_scale, torch.cat([scaled, tile_cond], dim=1), cnoise)
                mo = scale_score(mo, samples, sigma, sch.sigma_data, score_scaling)
                samples = sch.step(mo, t, samples)
            accumulate(out, out_w, samples, weights, i0, j0)
    return normalise(out, out_w)


def process_cond_img(cond_img, histogram_raw, cond_means, cond_stds, noise_level):
    """sample_diffusion_base.py:11-48, including its NaN handling of batch rows 0 and 1 and the unseeded randn fill
    of NaN climate means."""
    m = torch.as_tensor(cond_means)
    s = torch.as_tensor(cond_stds)
    x = (cond_img - m.view(1, -1, 1, 1)) / s.view(1, -1, 1, 1)
    x[0:1] = x[0:1].nan_to_num(float(m[0]))
    x[1:2] = x[1:2].nan_to_num(float(m[1]))
    noise_level = (torch.as_tensor(noise_level) - 0.5) * np.sqrt(12)
    clim = x[:, 2:6, 1:3, 1:3].mean(dim=(2, 3))
    clim[torch.isnan(clim)] = torch.randn_like(clim[torch.isnan(clim)])
    parts = [x[:, 0:1].flatten(1), x[:, 1:2].flatten(1), clim.flatten(1), x[:, 6:7].flatten(1), histogram_raw,
             noise_level.view(-1, 1)]
    return mp_concat(parts, [1.0 / len(parts)] * len(parts), dim=1).float()


@torch.no_grad()
def sample_base_diffusion(model_fn, make_scheduler, shape, cond_inputs, *, cond_means, cond_stds, noise_level,
                          histogram_raw, steps, noise, guide_fn=None, guidance_scale=1.0, tile_size=None):
    """model_fn / guide_fn(x[N,5,h,w], noise_labels[N], conditional_inputs) -> [N,5,h,w]; `noise` is the initial
    noise already multiplied by sigma_0 (the reference draws it with torch.randn(shape, generator) * sigma0)."""
    if tile_size is None:
        sch = make_scheduler()
        sch.set_timesteps(steps)
        samples = noise
        for t, sigma in zip(sch.timesteps, sch.sigmas):
            scaled = sch.precondition_inputs(samples, sigma)
            cnoise = sch.trigflow_precondition_noise(sigma.view(-1).expand(samples.shape[0]))
            mo = guided(model_fn, guide_fn, guidance_scale, scaled, cnoise, cond_inputs)
            samples = sch.step(mo, t, samples)
        return samples
    B, C, H, W = shape
    stride = tile_size // 2
    out = torch.zeros(shape)
    out_w = torch.zeros(shape)
    weights = linear_weight_window(tile_size)[None, None]
    for ic, i0 in enumerate(tile_starts(H, tile_size, stride)):
        for jc, j0 in enumerate(tile_starts(W, tile_size, stride)):
            tile_cond = [process_cond_img(cond_inputs[..., ic:ic + 4, jc:jc + 4], histogram_raw, cond_means,
                                          cond_stds, noise_level)]
            x = noise[..., i0:i0 + tile_size, j0:j0 + tile_size]
            sch = make_scheduler()
            sch.set_timesteps(steps)
            for t, sigma in zip(sch.timesteps, sch.sigmas):
                scaled = sch.precondition_inputs(x, sigma)
                cnoise = sch.trigflow_precondition_noise(sigma.view(-1).expand(x.shape[0]))
                mo = guided(model_fn, guide_fn, guidance_scale, scaled, cnoise, tile_cond)
                x = sch.step(mo, t, x)
            accumulate(out, out_w, x, weights, i0, j0)
    return normalise(out, out_w) / sch.sigma_data
