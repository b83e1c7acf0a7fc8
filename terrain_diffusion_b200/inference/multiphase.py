"""Generic multi-phase InfiniteDiffusion: an N-step diffusion schedule split into phases at timestep thresholds, every
phase solved tile by tile and BLENDED before the next phase reads it -- the algorithm of the reference's canonical demo
(annotated_infinite_panorama.py:84-102 `build_timestep_ranges`, :176-226 initial / continuation phases on chained lazy
canvases) and of its dense restatement (evaluation/infinite_consistency.py:207-239), for any EDMUnet2D denoiser +
EDM DPM-Solver++ scheduler of this package.

  phase 0       tile input = the tile of the noise field (already scaled by sigma_0), steps i in range 0
  phase p > 0   tile input = (sum x*w / sum w) of phase p-1 over the tile, steps i in range p

Within a phase every tile is an independent fused sub-solve (`DiffusionSolve(step_range=...)`: one CUDA graph per batch
of tiles); the per-tile solver state is reset at every phase start, because the blended canvas carries no multistep
history.  Two forms: `sample_infinite_diffusion` on a bounded canvas (tile_starts geometry, like the reference's
`sample_*_tiled` functions) and `infinite_diffusion_canvases` as a chain of unbounded `LazyCanvas`es (window-index
geometry, like the demo's chain of InfiniteTensors).
"""
from __future__ import annotations

import torch

from .lazy_canvas import LazyCanvas, TensorWindow
from .noise import gaussian_noise_patch
from .samplers import _blend_tiles, _gather, get_diffusion_solve
from .tiling import linear_weight_window, tile_starts


def build_timestep_ranges(all_timesteps: torch.Tensor, thresholds) -> list[torch.Tensor]:
    """Partition DESCENDING `all_timesteps` into phases (annotated_infinite_panorama.py:84-102): phase 0 gets
    t >= thresholds[0] (largest threshold first), the last phase gets t < the smallest threshold, empty ranges are
    dropped."""
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


def phase_step_ranges(scheduler, num_steps: int, thresholds) -> list[tuple[int, int]]:
    """(i0, i1) step-index ranges of the phases of an `num_steps` schedule, thresholds in the scheduler's timestep unit
    (`scheduler.timesteps`, descending: 0.25 * ln sigma for the EDM scheduler)."""
    scheduler.set_timesteps(num_steps)
    out, i = [], 0
    for r in build_timestep_ranges(scheduler.timesteps, thresholds):
        out.append((i, i + len(r)))
        i += len(r)
    assert i == num_steps
    return out


def pack(values_chw: torch.Tensor, weight_hw: torch.Tensor) -> torch.Tensor:
    """(C, H, W) + (H, W) -> (C+1, H, W) weighted window output (annotated_infinite_panorama.py:150-152)."""
    return torch.cat([values_chw * weight_hw[None], weight_hw[None]], dim=0)


def normalize(weighted: torch.Tensor) -> torch.Tensor:
    """(sum x*w, sum w) -> weighted average (annotated_infinite_panorama.py:147-148)."""
    return weighted[:-1] / weighted[-1:].clamp(min=1e-6)


@torch.no_grad()
def sample_infinite_diffusion(model, scheduler, cond_img: torch.Tensor, noise: torch.Tensor, tile_size: int,
                              tile_stride: int, *, num_steps: int, thresholds, tile_batch: int = 1) -> torch.Tensor:
    """Bounded canvas.  noise: [B, Cs, H, W] already scaled by sigma_0; cond_img: [B, Cc, H, W] or None.  Returns the
    blended result of the last phase, [B, Cs, H, W] (same convention as sample_decoder_diffusion_tiled)."""
    b, c, h, w = noise.shape
    device = noise.device
    window = linear_weight_window(tile_size, device).contiguous()
    tiles = [(i0, j0) for i0 in tile_starts(h, tile_size, tile_stride) for j0 in tile_starts(w, tile_size, tile_stride)]
    cond32 = None if cond_img is None else cond_img.to(device).float()
    current = noise.float()
    for rng in phase_step_ranges(scheduler, num_steps, thresholds):
        def run_group(chunk):
            solve = get_diffusion_solve(model, scheduler, b * len(chunk), tile_size, tile_size, num_steps,
                                        step_range=rng)
            cd = None if cond32 is None else _gather(cond32, chunk, tile_size)
            return solve.run(_gather(current, chunk, tile_size), cd)

        current = _blend_tiles(tiles, tile_batch, b, c, h, w, window, run_group)     # what the next phase reads
    return current.to(noise.dtype)


def infinite_diffusion_canvases(model, scheduler, seed: int, *, channels: int, tile_size: int, tile_stride: int,
                                num_steps: int, thresholds, cond_fn=None, batch_size: int | None = None,
                                cache_limit: int | None = None, noise_tile: int = 256) -> list[LazyCanvas]:
    """Unbounded form: one LazyCanvas per phase, chained like the demo's InfiniteTensors
    (annotated_infinite_panorama.py:204-226).  Window (0, i, j) covers rows [i*stride, i*stride + tile) etc.; the
    noise field is the tile-seeded one of the product pipeline (world_pipeline.py:66-115) scaled by sigma_0;
    `cond_fn(y0, x0, tile) -> [Cc, tile, tile]` supplies the conditioning channels of a window (None: unconditional
    model).  Returns the phase canvases, last one = the result; slice it and `normalize`."""
    dev = model.device
    ranges = phase_step_ranges(scheduler, num_steps, thresholds)
    sigma0 = float(scheduler.sigmas[0])
    win = TensorWindow((channels + 1, tile_size, tile_size), (channels + 1, tile_stride, tile_stride))
    weight = linear_weight_window(tile_size, dev).contiguous()

    def run_phase(rng, ctxs, inputs):
        solve = get_diffusion_solve(model, scheduler, len(ctxs), tile_size, tile_size, num_steps, step_range=rng)
        cd = None
        if cond_fn is not None:
            cd = torch.stack([cond_fn(i * tile_stride, j * tile_stride, tile_size).to(dev, torch.float32)
                              for (_, i, j) in ctxs])
        out = solve.run(torch.stack(inputs), cd)
        return [pack(out[k], weight) for k in range(len(ctxs))]

    def first(ctxs):
        single = not isinstance(ctxs, list)
        cl = [ctxs] if single else ctxs
        xs = [gaussian_noise_patch(seed, i * tile_stride, j * tile_stride, tile_size, tile_size, channels, noise_tile,
                                   noise_tile, device=dev) * sigma0 for (_, i, j) in cl]
        res = run_phase(ranges[0], cl, xs)
        return res[0] if single else res

    def later(rng):
        def f(ctxs, prev):
            single = not isinstance(ctxs, list)
            cl, pl = ([ctxs], [prev]) if single else (ctxs, prev)
            res = run_phase(rng, cl, [normalize(p.to(dev, torch.float32)) for p in pl])
            return res[0] if single else res
        return f

    canvases = [LazyCanvas(channels + 1, first, win, dev, batch_size=batch_size, cache_limit=cache_limit)]
    for rng in ranges[1:]:
        canvases.append(LazyCanvas(channels + 1, later(rng), win, dev, args=(canvases[-1],), args_windows=(win,),
                                   batch_size=batch_size, cache_limit=cache_limit))
    return canvases
