"""ORACLE (test infrastructure, not product): CPU restatement of the reference's tile dispatch and overlap blend.

Reference (xandergos/terrain-diffusion @ 82a0431):
  _tile_starts / _linear_weight_window          terrain_diffusion/training/evaluation/__init__.py:3-22
  linear_weight_window                          terrain_diffusion/inference/world_pipeline.py:117-124
  sample_decoder_diffusion_tiled                terrain_diffusion/training/evaluation/sample_diffusion_decoder.py:44-125
     (single-tile as written; multi-tile with the per-tile scheduler reset of sample_diffusion_base.py:147, because
      the function as shipped never resets the stateful scheduler between tiles -- SURVEY.md section 0 item 7)
  sample_decoder_consistency_tiled              .../sample_diffusion_decoder.py:129-211
  multi-phase consistency blend                 terrain_diffusion/evaluation/infinite_consistency.py:207-239
  window-index rule of the (external) infinite_tensor canvas, black-box from call sites
                                                world_pipeline.py:917-920,1091,1147,1230,1259-1260 (SURVEY App. C)

The third-party `infinite-tensor>=0.3.0` (requirements.txt:32) is absent from the reference checkout; its only arithmetic on
this path is "sum overlapping windows into an fp32 canvas, divide by the summed weight on read"
(annotated_infinite_panorama.py:141-146), restated here as accumulate()/normalise().  PARITY UNPINNED for that
library itself (no golden vectors exist); the bounded-canvas functions above ARE pinned against the reference by
tests/golden/make_golden.py.
"""
from __future__ import annotations

import math

import torch


def tile_starts(length: int, tile_size: int, stride: int) -> list[int]:
    if length <= tile_size:
        return [0]
    starts = list(range(0, max(1, length - tile_size + 1), max(1, stride)))
    if starts[-1] != length - tile_size:
        starts.append(length - tile_size)  # last tile clamped to the edge
    return starts


def linear_weight_window(size: int, dtype=torch.float32) -> torch.Tensor:
    """[size, size]: (1 - 0.999*|y-m|/m)(1 - 0.999*|x-m|/m), m = (size-1)/2, in the reference's op order."""
    mid = (size - 1) / 2
    y, x = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
    eps = 1e-3
    wy = 1 - (1 - eps) * torch.clamp(torch.abs(y - mid).to(dtype) / mid, 0, 1)
    wx = 1 - (1 - eps) * torch.clamp(torch.abs(x - mid).to(dtype) / mid, 0, 1)
    return wy * wx


def window_range(a: int, b: int, size: int, stride: int, offset: int = 0) -> range:
    """Indices k of windows [k*stride+offset, k*stride+offset+size) that intersect [a, b) (unbounded canvas;
    negative coordinates are real coordinates, floor semantics)."""
    k_lo = math.floor((a - offset - size) / stride) + 1
    k_hi = math.ceil((b - offset) / stride) - 1
    return range(k_lo, k_hi + 1)


def accumulate(canvas_val, canvas_w, tile, weights, i0, j0):
    """canvas[C] += x*w ; canvas[w] += w  (sample_diffusion_decoder.py:122-123)."""
    t = tile.shape[-1]
    canvas_val[..., i0:i0 + t, j0:j0 + t] += tile * weights
    canvas_w[..., i0:i0 + t, j0:j0 + t] += weights


def normalise(canvas_val, canvas_w):
    return canvas_val / canvas_w


@torch.no_grad()
def sample_decoder_diffusion_tiled(model_fn, make_scheduler, cond_img, noise, tile_size=None, tile_stride=None,
                                   num_steps=20):
    """model_fn(x[N,5,h,w], noise_labels[N]) -> [N,1,h,w];  make_scheduler() -> object with the reference scheduler
    surface (oracle.scheduler.OracleScheduler).  Sequential row-major tile order, fp32."""
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
                mo = model_fn(torch.cat([scaled, tile_cond], dim=1), cnoise)
                samples = sch.step(mo, t, samples)
            accumulate(out, out_w, samples, weights, i0, j0)
    return normalise(out, out_w)


@torch.no_grad()
def sample_decoder_consistency_tiled(model_fn, sigma_data, sigma0, cond_img, noise, tile_size=None, tile_stride=None,
                                     intermediate_t=()):
    b, c, h, w = noise.shape
    tile_size = tile_size or min(h, w)
    tile_stride = tile_stride or tile_size
    weights = linear_weight_window(tile_size, noise.dtype)[None, None]
    out = torch.zeros_like(noise)
    out_w = torch.zeros_like(noise)
    init_t = torch.atan(torch.as_tensor(sigma0 / sigma_data, dtype=noise.dtype))
    ts = (init_t, *[torch.tensor(t, dtype=noise.dtype) for t in intermediate_t])
    for i0 in tile_starts(h, tile_size, tile_stride):
        for j0 in tile_starts(w, tile_size, tile_stride):
            samples = torch.zeros((b, c, tile_size, tile_size), dtype=noise.dtype)
            tile_cond = cond_img[..., i0:i0 + tile_size, j0:j0 + tile_size]
            z = noise[..., i0:i0 + tile_size, j0:j0 + tile_size] * sigma_data
            for ts_ in ts:
                t = ts_.view(1, 1, 1, 1).expand(b, 1, 1, 1)
                x_t = torch.cos(t) * samples + torch.sin(t) * z
                pred = -model_fn(torch.cat([x_t / sigma_data, tile_cond], dim=1), t.flatten())
                samples = torch.cos(t) * x_t - torch.sin(t) * sigma_data * pred
            accumulate(out, out_w, samples, weights, i0, j0)
    return normalise(out, out_w) / sigma_data


# ---------------------------------------------------------------------------------------------- multi-phase
def build_timestep_ranges(all_timesteps: torch.Tensor, thresholds) -> list:
    """annotated_infinite_panorama.py:84-102: descending timesteps split at the (descending-sorted) thresholds."""
    thresholds = sorted(thresholds, reverse=True)
    if not thresholds:
        return [all_timesteps]
    ranges, prev = [], None
    for t in thresholds:
        r = all_timesteps[all_timesteps >= t] if prev is None else \
            all_timesteps[(all_timesteps >= t) & (all_timesteps < prev)]
        if len(r) > 0:
            ranges.append(r)
        prev = t
    tail = all_timesteps[all_timesteps < thresholds[-1]]
    if len(tail) > 0:
        ranges.append(tail)
    return ranges


@torch.no_grad()
def sample_infinite_diffusion(model_fn, make_scheduler, cond_img, noise, tile_size, tile_stride, num_steps, thresholds):
    """Dense multi-phase InfiniteDiffusion on a bounded canvas, fp32: the phase structure of
    annotated_infinite_panorama.py:176-226 (initial phase from the noise field, continuation phases from the BLENDED
    previous phase) in the loop shape of evaluation/infinite_consistency.py:207-239 (per phase: all tiles row-major ->
    weighted sum -> divide), with the diffusion step of sample_diffusion_decoder.py:105-120 inside and a per-tile
    scheduler reset at every phase start (no multistep history survives the blend).  noise is already scaled by
    sigma_0."""
    b, c, h, w = noise.shape
    weights = linear_weight_window(tile_size, noise.dtype)[None, None]
    probe = make_scheduler()
    probe.set_timesteps(num_steps)
    sample = noise
    i0s = 0
    for rng in build_timestep_ranges(probe.timesteps, thresholds):
        out = torch.zeros_like(noise)
        out_w = torch.zeros_like(noise)
        for i0 in tile_starts(h, tile_size, tile_stride):
            for j0 in tile_starts(w, tile_size, tile_stride):
                sch = make_scheduler()
                sch.set_timesteps(num_steps)
                sch.step_index = i0s                      # positioned at the phase's first step, empty history
                x = sample[..., i0:i0 + tile_size, j0:j0 + tile_size]
                tc = cond_img[..., i0:i0 + tile_size, j0:j0 + tile_size]
                for k in range(i0s, i0s + len(rng)):
                    sigma = sch.sigmas[k]
                    scaled = sch.precondition_inputs(x, sigma)
                    cnoise = sch.trigflow_precondition_noise(sigma.view(-1).expand(b))
                    x = sch.step(model_fn(torch.cat([scaled, tc], dim=1), cnoise), sch.timesteps[k], x)
                accumulate(out, out_w, x, weights, i0, j0)
        sample = normalise(out, out_w)
        i0s += len(rng)
    return sample
