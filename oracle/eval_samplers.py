"""ORACLE (test infrastructure, not product): fp32 CPU restatement of the reference's consistency-base and coarse
evaluation samplers.

Reference (xandergos/terrain-diffusion @ 82a0431):
  sample_base_consistency                       terrain_diffusion/training/evaluation/sample_diffusion_base.py:171-268
  _cond_inputs_from_snr / sample_coarse_tiled   terrain_diffusion/training/evaluation/sample_coarse.py:7-125

Pinned against the reference by tests/golden/make_golden_eval.py.  The coarse sampler is restated with a scheduler
reset per tile (the shipped function fails on a second tile, SURVEY.md section 0 item 7); the golden uses one tile,
where both agree.
"""
from __future__ import annotations

import torch

from .guided import process_cond_img
from .tiling import accumulate, linear_weight_window, normalise, tile_starts


@torch.no_grad()
def sample_base_consistency(model_fn, sigma0, sigma_data, shape, cond_inputs, *, cond_means, cond_stds, noise_level,
                            histogram_raw, intermediate_t, tile_size, noise):
    """model_fn(x[N,5,h,w], noise_labels[N], conditional_inputs) -> [N,5,h,w]; noise[k]: the unit noise of phase k."""
    B, C, H, W = shape
    stride = tile_size // 2
    ts = [torch.atan(torch.as_tensor(sigma0, dtype=torch.float32) / sigma_data)]
    if intermediate_t > 0:
        ts.append(torch.tensor(intermediate_t, dtype=torch.float32))
    weights = linear_weight_window(tile_size)[None, None]
    sample = torch.zeros(shape)
    for k, t_s in enumerate(ts):
        out = torch.zeros(shape)
        out_w = torch.zeros(shape)
        for ic, i0 in enumerate(tile_starts(H, tile_size, stride)):
            for jc, j0 in enumerate(tile_starts(W, tile_size, stride)):
                if cond_inputs.ndim == 4:
                    tile_cond = [process_cond_img(cond_inputs[..., ic:ic + 4, jc:jc + 4], histogram_raw, cond_means,
                                                  cond_stds, noise_level)]
                else:
                    tile_cond = [cond_inputs]
                z = noise[k][..., i0:i0 + tile_size, j0:j0 + tile_size] * sigma_data
                s = sample[..., i0:i0 + tile_size, j0:j0 + tile_size]
                t = t_s.view(1, 1, 1, 1).expand(B, 1, 1, 1)
                x_t = torch.cos(t) * s + torch.sin(t) * z
                pred = -model_fn(x_t / sigma_data, t.flatten(), tile_cond)
                accumulate(out, out_w, torch.cos(t) * x_t - torch.sin(t) * sigma_data * pred, weights, i0, j0)
        sample = normalise(out, out_w)
    return sample / sigma_data


def cond_inputs_from_snr(cond_snr):
    """[1, 5] SNR -> five [1] float conditions log(tan(atan(snr)) / 8)."""
    vals = torch.log(torch.tan(torch.atan(cond_snr)) / 8.0)
    return [v.view(-1) for v in vals.transpose(0, 1)]


@torch.no_grad()
def sample_coarse_tiled(model_fn, make_scheduler, cond_img, cond_snr, *, steps, tile_size, tile_stride, out_channels,
                        cond_noise, tile_noise):
    """model_fn(x[N,11,h,w], noise_labels[N], conditional_inputs) -> [N,6,h,w].  cond_noise: the randn_like(cond_img)
    draw; tile_noise[k]: the unit noise of tile k in row-major order (the reference multiplies it by sigma_0)."""
    b, _, h, w = cond_img.shape
    weights = linear_weight_window(tile_size)[None, None]
    out = torch.zeros((b, out_channels, h, w))
    out_w = torch.zeros_like(out)
    cond = cond_inputs_from_snr(cond_snr)
    t_cond = torch.atan(cond_snr).view(1, -1, 1, 1)
    cond_img = torch.cos(t_cond) * cond_img + torch.sin(t_cond) * cond_noise
    k = 0
    for i0 in tile_starts(h, tile_size, tile_stride):
        for j0 in tile_starts(w, tile_size, tile_stride):
            sch = make_scheduler()
            sch.set_timesteps(steps)
            x = tile_noise[k] * sch.sigmas[0]
            k += 1
            tc = cond_img[..., i0:i0 + tile_size, j0:j0 + tile_size]
            for t, sigma in zip(sch.timesteps, sch.sigmas):
                scaled = sch.precondition_inputs(x, sigma)
                cnoise = sch.trigflow_precondition_noise(sigma.view(-1).expand(b))
                x = sch.step(model_fn(torch.cat([scaled, tc], dim=1), cnoise, cond), t, x)
            accumulate(out, out_w, x / sch.sigma_data, weights, i0, j0)
    return normalise(out, out_w)
