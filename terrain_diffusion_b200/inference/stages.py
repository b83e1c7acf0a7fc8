"""The three InfiniteDiffusion stages of the product pipeline as device programs.

What the reference does per tile in `WorldPipeline._coarse_inference / _latent_inference / _decoder_inference`
(inference/world_pipeline.py:909-959, 1052-1131, 1209-1242) -- numba noise on the CPU, H2D, a dozen small torch ops
around the U-Net, `.item()`, D2H -- is organised here around ONE fused program per batch of tiles:

  consistency stages   `get_consistency_solve`: first convolution reads (sample * c_in | conditioning), the U-Net runs as
                       a CUDA graph, the LAST convolution applies the TrigFlow update s' = cos t x_t + sin t sigma_d F
                       (and the final 1 / sigma_d).  A first phase starts from s = 0, so x_t = sin t sigma_d z folds into
                       the two scalars and the noise tile goes straight into the sample buffer; a later phase needs one
                       mixing launch (tdx_trig_mix).  The packed window output cat([x w, w]) is one launch
                       (tdx_pack_weighted); normalise-on-read + nearest upsampling of the latent window one launch
                       (tdx_window_to_cond).
  coarse stage         `get_diffusion_solve`: the 20-step DPM-Solver++ solve as one graph, the embeddings of all steps
                       from one batched call.

Noise comes from the bit-compatible GPU generator (same seeds as the reference), nothing synchronises with the host and
nothing leaves the GPU.  Taken as arguments, because the reference computes them outside the hot path: the synthetic
conditioning map of the coarse stage and the blended dependency windows the canvas engine hands to each callback.
"""
from __future__ import annotations

import math

import torch

from .. import _lib as L
from .noise import gaussian_noise_patch, gaussian_noise_patches
from .samplers import get_consistency_solve, get_diffusion_solve
from .tiling import padded_batch_size

LATENT_TILE, LATENT_STRIDE = 64, 32          # world_pipeline.py:1054-1055
COARSE_TILE, COARSE_STRIDE = 64, 48          # world_pipeline.py:913-914


# ------------------------------------------------------------------------------------------------ launches
def _f32(t: torch.Tensor, dev) -> torch.Tensor:
    return t.to(device=dev, dtype=torch.float32).contiguous()


def trig_mix(sample, noise: torch.Tensor, a: float, b: float) -> torch.Tensor:
    """a * sample + b * noise in one launch (sample None: zeros)."""
    out = torch.empty_like(noise)
    L.call(L.lib().tdx_trig_mix, noise.device, out.data_ptr(), None if sample is None else sample.data_ptr(),
           noise.data_ptr(), noise.numel(), float(a), float(b))
    return out


def pack_weighted(x: torch.Tensor, window: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """[n, C, T, T] -> [n, C+1, T, T] = cat([x * scale * w, w]): the packed window output of every stage."""
    n, c, h, w = x.shape
    out = torch.empty((n, c + 1, h, w), dtype=torch.float32, device=x.device)
    L.call(L.lib().tdx_pack_weighted, x.device, out.data_ptr(), x.data_ptr(), window.data_ptr(), n, c, h * w,
           float(scale))
    return out


def window_to_cond(packed: torch.Tensor, keep: int, factor: int) -> torch.Tensor:
    """[n, C+1, h, w] packed window -> [n, keep, h*factor, w*factor]: (sum x w / sum w), nearest-upsampled."""
    n, cp, h, w = packed.shape
    out = torch.empty((n, keep, h * factor, w * factor), dtype=torch.float32, device=packed.device)
    L.call(L.lib().tdx_window_to_cond, packed.device, out.data_ptr(), packed.data_ptr(), n, cp, keep, h, w, factor)
    return out


# ------------------------------------------------------------------------------------------------ decoder stage
@torch.no_grad()
def decoder_stage_tile(model, seed: int, ctx, latents: torch.Tensor, weight_window: torch.Tensor, t_list,
                       tile_size: int = 512, tile_stride: int = 384, sigma_data: float = 0.5,
                       latent_compression: int = 8) -> torch.Tensor:
    """Decoder window (0, i, j): packed [6, T/lc, T/lc] latent window in, packed [2, T, T] residual window out
    (world_pipeline.py:1209-1242; one consistency step per entry of t_list, product: a single step at t_init)."""
    dev = model.device
    T = tile_size
    cond = window_to_cond(_f32(latents, dev)[None], 4, latent_compression)
    sample = None
    for k, t in enumerate(t_list):
        t = float(t)
        z = gaussian_noise_patch(seed + 5819 + k, ctx[1] * tile_stride, ctx[2] * tile_stride, T, T, 1, T, T,
                                 device=dev)[None]
        last = k == len(t_list) - 1
        solve = get_consistency_solve(model, 1, T, T, t, sigma_data, from_unit_noise=(k == 0),
                                      out_scale=1.0 / sigma_data if last else 1.0)
        x = z if k == 0 else trig_mix(sample, z, math.cos(t), math.sin(t) * sigma_data)
        sample = solve.run(x, cond)
    return pack_weighted(sample, _f32(weight_window, dev))[0]


# ------------------------------------------------------------------------------------------------ latent stage
_DEV_CONSTS: dict = {}


def _const_on(dev, t) -> torch.Tensor:
    """fp32 device copy of a small HOST constant (statistics vectors, histogram, noise level), cached by CONTENT: every
    stage call passes the same few values, and each pageable `.to(device)` is a blocking copy (these copies were half
    of the host time of a cold `WorldPipeline.get`)."""
    t = torch.as_tensor(t)
    if t.device.type != "cpu" or t.numel() > 4096:
        return t.to(device=dev, dtype=torch.float32)
    t = t.detach().to(torch.float32).contiguous()
    key = (str(dev), tuple(t.shape), t.numpy().tobytes())
    hit = _DEV_CONSTS.get(key)
    if hit is None:
        if len(_DEV_CONSTS) > 256:
            _DEV_CONSTS.clear()
        hit = _DEV_CONSTS[key] = t.clone().to(dev)      # (clone: on a CPU `dev` .to() would alias the caller's tensor)
    return hit


def _concat_scales(dims, dev) -> torch.Tensor:
    """mp_concat with equal weights (mp_layers.py:65-86) as ONE per-column scale vector: part i of width N_i is
    multiplied by sqrt(sum N / sum w^2) / sqrt(N_i) * w_i with w_i = 1 / len(parts)."""
    k = len(dims)
    c = math.sqrt(sum(dims) / (k * (1.0 / k) ** 2))
    return _const_on(dev, torch.cat([torch.full((d,), c / math.sqrt(d) / k, dtype=torch.float32) for d in dims]))


@torch.no_grad()
def process_latent_conditioning(cond_img, histogram_raw, cond_means, cond_stds, noise_level, seed=0, seed_offset=0,
                                reference_sampler_nans: bool = False):
    """The 58-dim condition vector of the base model for a batch of coarse windows (world_pipeline.py:1018-1050):
    cond_img [n, 7, 4, 4] = de-blended coarse channels + mask.  Batched, on cond_img's device, no host round trip.
    The reference replaces every NaN of its batch-of-one tensor by cond_means[0] before it looks for NaNs in the climate
    crop, so its seeded NaN fill (:1040-1044) can never trigger; `seed` / `seed_offset` are accepted for signature
    compatibility.  histogram_raw is [H] (shared) or [n, H] (per row); noise_level a scalar, [1] or [n, 1].
    reference_sampler_nans: the NaN handling of the evaluation sampler's `_process_cond_img`
    (sample_diffusion_base.py:36-46) instead: NaNs of batch ROW 0 become cond_means[0], of row 1 cond_means[1], and
    NaN climate means are filled with unseeded standard normals (SURVEY Appendix G)."""
    dev = cond_img.device
    n = cond_img.shape[0]
    cond_means = torch.as_tensor(cond_means)
    x = (cond_img.float() - _const_on(dev, cond_means).view(1, -1, 1, 1)) / _const_on(dev, cond_stds).view(1, -1, 1, 1)
    if reference_sampler_nans:
        cm = cond_means.flatten()
        x[0:1] = torch.nan_to_num(x[0:1], nan=float(cm[0]))
        x[1:2] = torch.nan_to_num(x[1:2], nan=float(cm[1]))
    else:
        x = torch.nan_to_num(x, nan=float(cond_means.flatten()[0]))
    level = _const_on(dev, ((torch.as_tensor(noise_level, dtype=torch.float32).cpu() - 0.5) * math.sqrt(12)).reshape(-1, 1))
    hist = _const_on(dev, histogram_raw)
    hist = hist.reshape(1, -1) if hist.dim() < 2 else hist
    clim = x[:, 2:6, 1:3, 1:3].mean(dim=(2, 3))
    if reference_sampler_nans:
        bad = torch.isnan(clim)
        clim[bad] = torch.randn_like(clim[bad])
    parts = [x[:, 0].flatten(1), x[:, 1].flatten(1), clim, x[:, 6].flatten(1),
             hist.expand(n, -1), level.expand(n, -1)]
    return torch.cat(parts, dim=1) * _concat_scales([p.shape[1] for p in parts], dev)


@torch.no_grad()
def latent_stage_tiles(model, seed: int, ctxs, samples, cond_imgs, t: float, weight_window: torch.Tensor,
                       histogram_raw, cond_means, cond_stds, seed_offset: int = 0, sigma_data: float = 0.5,
                       pad_batch_to=None) -> list:
    """One consistency phase of the latent stage for a batch of window indices (world_pipeline.py:1052-1131).
    samples: None (first phase) or packed [6, 64, 64] windows of the previous phase's canvas; cond_imgs: packed
    [7, 4, 4] coarse windows.  Returns the packed [6, 64, 64] tiles (views of one device tensor)."""
    if not ctxs:
        return []
    dev = model.device
    n, T = len(ctxs), LATENT_TILE
    t = float(t)
    cond_imgs = [torch.as_tensor(c) for c in cond_imgs]
    if all(c.device.type == "cpu" for c in cond_imgs):            # host windows (the reference's convention): ONE copy
        coarse = _f32(torch.stack(cond_imgs), dev)
    else:
        coarse = torch.stack([_f32(c, dev) for c in cond_imgs])                                  # [n, 7, 4, 4] packed
    cimg = torch.cat([coarse[:, :-1] / coarse[:, -1:], torch.ones((n, 1, 4, 4), device=dev)], dim=1)
    cvec = process_latent_conditioning(cimg, histogram_raw, cond_means, cond_stds, torch.tensor(0.0))
    z = gaussian_noise_patches(seed + seed_offset, [(c[1] * LATENT_STRIDE, c[2] * LATENT_STRIDE) for c in ctxs], T, T, 5,
                               T, T, device=dev)
    first = samples is None or all(s is None for s in samples)
    if first:
        x = z                                                   # s = 0: x_t = sin t sigma_d z, folded into the program
    else:
        prev = torch.stack([_f32(torch.as_tensor(s), dev) for s in samples])                     # [n, 6, T, T] packed
        x = trig_mix(window_to_cond(prev, 5, 1), z, math.cos(t) * sigma_data, math.sin(t) * sigma_data)
    m = padded_batch_size(n, pad_batch_to) if pad_batch_to else n
    if m > n:   # the reference pads to {1,2,4,8,16} under torch.compile (:393-398, 1107-1118): one plan per size
        x = torch.cat([x, x[:1].expand(m - n, -1, -1, -1)], dim=0)
        cvec = torch.cat([cvec, cvec[:1].expand(m - n, -1)], dim=0)
    solve = get_consistency_solve(model, m, T, T, t, sigma_data, from_unit_noise=first, out_scale=1.0 / sigma_data)
    sample = solve.run(x, None, conditional_inputs=[cvec])
    return list(pack_weighted(sample[:n], _f32(weight_window, dev)))


# ------------------------------------------------------------------------------------------------ coarse stage
@torch.no_grad()
def coarse_stage_tile(model, scheduler, seed: int, ctx, synthetic_map: torch.Tensor, t_cond: torch.Tensor,
                      cond_inputs, weight_window: torch.Tensor, coarse_means, coarse_stds, num_steps: int = 20,
                      pool_size: int = 1) -> torch.Tensor:
    """Coarse window (0, i, j): 20-step DPM-Solver++ solve conditioned on the noised synthetic map
    (world_pipeline.py:909-959).  synthetic_map: the raw [5, 64, 64] conditioning of this window (built by the
    reference's Perlin / WorldClim machinery, out of scope).  Returns the packed [7, 64, 64] tile."""
    if pool_size != 1:
        raise NotImplementedError("coarse_pooling > 1 is host-side pooling of the finished tile; not on the GPU path")
    dev = model.device
    T = COARSE_TILE
    y0, x0 = ctx[1] * COARSE_STRIDE, ctx[2] * COARSE_STRIDE
    means = _const_on(dev, torch.as_tensor(coarse_means, dtype=torch.float32))
    stds = _const_on(dev, torch.as_tensor(coarse_stds, dtype=torch.float32))
    sel = [0, 2, 3, 4, 5]                                        # model statistics of the map's five channels (:925)
    smap = (_f32(synthetic_map, dev) - means[sel, None, None]) / stds[sel, None, None]
    tc = _const_on(dev, t_cond).view(-1, 1, 1)
    cond = (torch.cos(tc) * smap + torch.sin(tc) * gaussian_noise_patch(seed, y0, x0, T, T, 5, T, T, device=dev))[None]
    solve = get_diffusion_solve(model, scheduler, 1, T, T, num_steps)
    noise = gaussian_noise_patch(seed + 1, y0, x0, T, T, 6, T, T, device=dev)[None]
    sample = solve.run(noise * float(scheduler.sigmas[0]), cond,
                       conditional_inputs=[_const_on(dev, c) for c in cond_inputs])
    out = sample / float(scheduler.config.sigma_data) * stds.view(1, -1, 1, 1) + means.view(1, -1, 1, 1)
    out[:, 1] = out[:, 0] - out[:, 1]                            # channel 1 is predicted as (ch0 - ch1) (:953)
    return pack_weighted(out.contiguous(), _f32(weight_window, dev))[0]
