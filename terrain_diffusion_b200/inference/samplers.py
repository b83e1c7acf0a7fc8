"""Bounded-canvas tiled samplers -- drop-ins for terrain_diffusion.training.evaluation.sample_diffusion_decoder
(reference sample_diffusion_decoder.py:44-211), .sample_diffusion_base and .sample_coarse, running tile solves as
fused CUDA graphs and the overlap blend on a device-resident canvas.

Tile order, tile origins (`tile_starts`, last tile clamped) and the blend window are the reference's, integer for
integer.  Unlike the reference function as shipped, the multi-tile diffusion sampler resets the solver state per tile
(the reference raises IndexError on tile #2 because its stateful scheduler is never reset -- SURVEY.md section 0
item 7); the per-tile reset is the behaviour of the reference's own working samplers (sample_diffusion_base.py:147,
world_pipeline.py:934).  Independent tiles may be solved `tile_batch` at a time; the blend is still applied in
row-major order so the canvas is bit-identical to a sequential run.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from .canvas import BlendCanvas
from .solve import DiffusionSolve
from .tiling import linear_weight_window, tile_starts


MAX_CACHED_SOLVES = 12      # every cached solve owns an activation arena and a CUDA graph


class _LruDict(dict):
    """dict that keeps at most MAX_CACHED_SOLVES entries, dropping the least recently inserted / fetched."""

    def __getitem__(self, k):
        v = super().pop(k)
        super().__setitem__(k, v)
        return v

    def __setitem__(self, k, v):
        super().__setitem__(k, v)
        while len(self) > MAX_CACHED_SOLVES:
            super().pop(next(iter(self)))


def _solve_cache(model):
    if not hasattr(model, "_solve_cache"):
        model._solve_cache = _LruDict()
    return model._solve_cache


def get_diffusion_solve(model, scheduler, n, h, w, num_steps, step_range=None, guide=None, guidance_scale: float = 1.0,
                        score_scaling: float = 1.0, batch_invariant: bool = False) -> DiffusionSolve:
    """Cached fused N-step solve (or one phase of it: step_range).  The key is everything the solve bakes in: the
    sigma table and the per-step order schedule (they cover sigma_min/max/rho/schedule, scaling_p/scaling_t,
    lower_order_final, euler_at_final, ...) plus the options that change the update formula, and for a guided solve
    the guide's weights, the guidance scale and the score scaling.  The caller's scheduler is put in the state the
    reference leaves it in (`set_timesteps(num_steps)`) on a cache hit too.  batch_invariant: see DiffusionSolve."""
    scheduler.set_timesteps(num_steps)
    c = scheduler.config
    key = (n, h, w, num_steps, None if step_range is None else tuple(int(v) for v in step_range),
           tuple(float(v) for v in scheduler.sigmas), tuple(scheduler.order_schedule()),
           float(c.sigma_data), c.prediction_type, c.final_sigmas_type, c.solver_order, c.algorithm_type, c.solver_type,
           id(model.folded()))
    guided = guide is not None and float(guidance_scale) != 1.0
    if guided:
        key += ("guide", id(guide.folded()), float(guidance_scale))
    if score_scaling != 1.0:
        key += ("score_scaling", float(score_scaling))
    if batch_invariant:
        key += ("batch_invariant",)
    cache = _solve_cache(model)
    if key not in cache:
        cache[key] = DiffusionSolve(model, scheduler, n, h, w, num_steps, step_range=step_range,
                                    guide=guide if guided else None, guidance_scale=guidance_scale,
                                    score_scaling=score_scaling, batch_invariant=batch_invariant)
    return cache[key]


def get_consistency_solve(model, n, h, w, t: float, sigma_data: float = 0.5, from_unit_noise: bool = False,
                          out_scale: float = 1.0, batch_invariant: bool = False,
                          plan_images: int = 1) -> DiffusionSolve:
    """Cached one-step TrigFlow consistency program (solve.consistency_rows) for `n` tiles of h x w.
    batch_invariant, plan_images: see DiffusionSolve."""
    from .solve import consistency_rows
    key = ("cm", n, h, w, float(t), float(sigma_data), bool(from_unit_noise), float(out_scale), id(model.folded()))
    if plan_images != 1:
        key += ("plan_images", int(plan_images))
    if batch_invariant:
        key += ("batch_invariant",)
    cache = _solve_cache(model)
    if key not in cache:
        cache[key] = DiffusionSolve(model, None, n, h, w, 1,
                                    coef_rows=consistency_rows(t, sigma_data, from_unit_noise, out_scale),
                                    batch_invariant=batch_invariant, plan_images=plan_images)
    return cache[key]


def _window(weight_window_fn, size: int, device) -> torch.Tensor:
    """[size, size] contiguous fp32 blend weights on `device`: weight_window_fn(size, device, dtype) ([size, size] or
    [1, 1, size, size], as the reference's window functions return) or the reference's linear window."""
    if weight_window_fn is None:
        return linear_weight_window(size, device).contiguous()
    w = weight_window_fn(size, device, torch.float32)
    return w.to(device=device, dtype=torch.float32).reshape(size, size).contiguous()


def _gather(x: torch.Tensor, chunk, size: int) -> torch.Tensor:
    """The size x size windows of x at the (i0, j0, ...) tiles of `chunk`, concatenated on the batch axis."""
    return torch.cat([x[..., i0:i0 + size, j0:j0 + size] for i0, j0, *_ in chunk], dim=0)


def _blend_tiles(tiles, tile_batch: Optional[int], b: int, channels: int, height: int, width: int,
                 window: torch.Tensor, run_group, divisor: float = 1.0) -> torch.Tensor:
    """Solve `tiles` (row-major tuples that start with the tile origin (i0, j0)) in groups of `tile_batch` (None: all
    in one group) and blend them in row-major order.  run_group(chunk) returns the chunk's outputs, [len(chunk) * b,
    C, T, T] fp32 with the b images of a tile adjacent.  The b images share one canvas of b * C planes: every plane is
    blended independently, so this is bit-identical to one canvas per image.  Returns the normalised [b, C, H, W]."""
    canvas = BlendCanvas(b * channels, height, width, window.device)
    t = window.shape[-1]
    group = len(tiles) if tile_batch is None else max(1, int(tile_batch))
    for g0 in range(0, len(tiles), group):
        chunk = tiles[g0:g0 + group]
        out = run_group(chunk)
        for q, (i0, j0, *_) in enumerate(chunk):
            canvas.accumulate(out[q * b:(q + 1) * b].reshape(b * channels, t, t), i0, j0, window)
    return canvas.normalized(divisor).view(b, channels, height, width)


@torch.no_grad()
def sample_decoder_diffusion_tiled(model, scheduler, cond_img: torch.Tensor, noise: torch.Tensor,
                                   tile_size: Optional[int] = None, tile_stride: Optional[int] = None, *,
                                   num_steps: Optional[int] = None, guidance_model=None, guidance_scale: float = 1.0,
                                   score_scaling: float = 1.0, weight_window_fn=None, tile_batch: int = 1):
    """guidance_model / guidance_scale: two-model guidance F = F_g + s*(F_m - F_g) inside the fused solve (both
    forwards and the combination in one graph; the guide must have multiples of 64 channels in every layer).
    score_scaling: the reference's EDM score scaling (`_scale_score`), folded into the step coefficients."""
    if num_steps is None:
        num_steps = scheduler.num_inference_steps
        if num_steps is None:
            raise ValueError("num_steps is None and scheduler.set_timesteps was never called")
    b, c, h, w = noise.shape
    device, dtype = noise.device, noise.dtype
    cond_img = cond_img.to(device=device, dtype=dtype)
    if cond_img.shape[-2:] != (h, w):
        cond_img = F.interpolate(cond_img, size=(h, w), mode="nearest")
    tile_size = tile_size or min(h, w)
    tile_stride = tile_stride or tile_size
    window = _window(weight_window_fn, tile_size, device)
    tiles = [(i0, j0) for i0 in tile_starts(h, tile_size, tile_stride) for j0 in tile_starts(w, tile_size, tile_stride)]
    noise32, cond32 = noise.float(), cond_img.float()

    def run_group(chunk):
        solve = get_diffusion_solve(model, scheduler, b * len(chunk), tile_size, tile_size, num_steps,
                                    guide=guidance_model, guidance_scale=guidance_scale, score_scaling=score_scaling)
        return solve.run(_gather(noise32, chunk, tile_size), _gather(cond32, chunk, tile_size))

    return _blend_tiles(tiles, tile_batch, b, c, h, w, window, run_group).to(dtype)


def _reference_cond_vector(tile_cond, histogram_raw, cond_means, cond_stds, noise_level):
    """sample_diffusion_base.py:11-48 (`_process_cond_img`) for one window: the NaN handling of the reference's
    evaluation sampler (batch ROWS 0 and 1, unseeded randn for NaN climate means) on top of the product's vector."""
    from .stages import process_latent_conditioning
    return process_latent_conditioning(tile_cond, histogram_raw, cond_means, cond_stds, noise_level,
                                       reference_sampler_nans=True)


def _base_tiles(cond_inputs, H: int, W: int, tile_size: int):
    """(cond_inputs as a tensor, tiles) of the tiled base samplers: tiles of stride tile_size // 2 as (i0, j0, ic, jc),
    where [ic:ic+4, jc:jc+4] is the tile's window of a 4-D condition image.  ValueError unless a condition image is
    (len(starts)+3)-sized, and for a 1-D condition vector on more than one tile."""
    stride = tile_size // 2
    h_starts, w_starts = tile_starts(H, tile_size, stride), tile_starts(W, tile_size, stride)
    cond_inputs = torch.as_tensor(cond_inputs)
    if cond_inputs.ndim == 1 and len(h_starts) * len(w_starts) > 1:
        raise ValueError(f"cond_inputs must be a tensor image for tiled sampling. Cond inputs must have width "
                         f"{len(w_starts)+3} and height {len(h_starts)+3}.")
    elif cond_inputs.ndim == 4:
        if cond_inputs.shape[-1] != len(w_starts) + 3 or cond_inputs.shape[-2] != len(h_starts) + 3:
            raise ValueError(f"cond_inputs is {tuple(cond_inputs.shape[-2:])}; tiled sampling of {H}x{W} needs "
                             f"{len(h_starts)+3}x{len(w_starts)+3}")
    return cond_inputs, [(i0, j0, ic, jc) for ic, i0 in enumerate(h_starts) for jc, j0 in enumerate(w_starts)]


@torch.no_grad()
def sample_base_diffusion(model, scheduler, shape, cond_inputs, *, cond_means, cond_stds, noise_level=0.0,
                          histogram_raw, dtype=torch.float32, steps: int = 15, guide_model=None,
                          guidance_scale: float = 1.0, generator: Optional[torch.Generator] = None,
                          tile_size: Optional[int] = None, weight_window_fn=None, tile_batch: Optional[int] = None):
    """The base model's diffusion sampler (training/evaluation/sample_diffusion_base.py:51-168), optionally with
    two-model guidance; every N-step solve is one fused graph (both models per step when guided).

    Untiled (tile_size None): `cond_inputs` is passed to the model as given (a list of conditional inputs) and the
    result is NOT divided by sigma_data.  Tiled: stride tile_size // 2; each tile's 58-dim condition vector comes from
    the [ic:ic+4, jc:jc+4] window of the (len(starts)+3)-sized cond image; each tile starts from a fresh solver; tiles
    are blended in row-major order and the result is divided by sigma_data.  Independent tiles are solved
    `tile_batch` at a time (default: all at once); the blend order, and so the result, does not depend on it.

    The initial noise is torch.randn(shape, generator=generator) * sigma_0 as the reference draws it; a CPU generator
    draws on the CPU and the noise is copied to the model's device."""
    device = model.device
    scheduler.set_timesteps(steps)
    sigma0 = float(scheduler.sigmas[0])      # sigma_max: the same for every step count
    gen_dev = generator.device if generator is not None else device
    noise = torch.randn(tuple(shape), generator=generator, device=gen_dev, dtype=dtype)
    noise = (noise * torch.tensor(sigma0, dtype=torch.float32).to(noise.device)).to(device)
    B, C, H, W = shape
    if tile_size is None:
        solve = get_diffusion_solve(model, scheduler, B, H, W, steps, guide=guide_model, guidance_scale=guidance_scale)
        out = solve.run(noise.float(), None, conditional_inputs=[torch.as_tensor(c).to(device) for c in cond_inputs])
        return out.clone().to(dtype)

    cond_inputs, grid = _base_tiles(cond_inputs, H, W, tile_size)
    window = _window(weight_window_fn, tile_size, device)
    # every tile carries its condition vector, computed in tile order (the reference computes them in this order too:
    # the unseeded NaN fill draws from the global generator one tile after the other)
    if cond_inputs.ndim == 4:
        cimg = cond_inputs.to(device)
        tiles = [(i0, j0, _reference_cond_vector(cimg[..., ic:ic + 4, jc:jc + 4], histogram_raw, cond_means, cond_stds,
                                                 noise_level)) for i0, j0, ic, jc in grid]
    else:
        fixed = cond_inputs.to(device).float().reshape(1, -1).expand(B, -1)
        tiles = [(i0, j0, fixed) for i0, j0, _, _ in grid]

    def run_group(chunk):
        solve = get_diffusion_solve(model, scheduler, B * len(chunk), tile_size, tile_size, steps, guide=guide_model,
                                    guidance_scale=guidance_scale)
        cv = torch.cat([cvec for _, _, cvec in chunk], dim=0)
        return solve.run(_gather(noise, chunk, tile_size).float(), None, conditional_inputs=[cv])

    sd = float(scheduler.config.sigma_data)
    return _blend_tiles(tiles, tile_batch, B, C, H, W, window, run_group, sd).to(dtype)


def _phase_times(scheduler, intermediate_t, dtype) -> list:
    """Consistency times as the reference's evaluation sampler forms them (sample_diffusion_base.py:216-220): the fp32
    atan(sigma_0 / sigma_d) cast to `dtype`, then intermediate_t if > 0; returned as the floats of those tensors."""
    sigma_data = float(scheduler.config.sigma_data)
    ts = [float(torch.atan(scheduler.sigmas[0] / sigma_data).to(dtype))]
    if intermediate_t > 0:
        ts.append(float(torch.tensor(intermediate_t, dtype=dtype)))
    return ts


@torch.no_grad()
def sample_base_consistency(model, scheduler, shape, cond_inputs, *, cond_means, cond_stds, noise_level=0.0,
                            histogram_raw, intermediate_t=0.0, dtype=torch.float32,
                            generator: Optional[torch.Generator] = None, tile_size: Optional[int] = None,
                            weight_window_fn=None, noise=None, tile_batch: Optional[int] = None):
    """The base consistency model's evaluation sampler (training/evaluation/sample_diffusion_base.py:171-268): one
    TrigFlow step per phase at t_0 = atan(sigma_0 / sigma_d), then at `intermediate_t` if > 0.

    Per phase: x_t = cos t * s + sin t * sigma_d * z per tile (s = 0 in the first phase, the previous phase's blended
    canvas after it), s' = cos t * x_t - sin t * sigma_d * pred with pred = -model(x_t / sigma_d, t, [cvec]), tiles of
    stride tile_size // 2 blended in row-major order and normalised; the result is divided by sigma_d.  Every phase
    of `tile_batch` tiles (default: all) is one fused consistency program (get_consistency_solve); the blend order,
    and so the canvas, does not depend on the grouping, the implicit-GEMM work split does (DESIGN section 2).

    z is noise[k] if given, else one torch.randn(shape, generator=generator) per phase, drawn on the generator's device
    before that phase's tiles and copied to the model's device.  A 4-D `cond_inputs` is the (len(starts)+3)-sized
    condition image: each tile's vector comes from its [ic:ic+4, jc:jc+4] window, recomputed every phase as the
    reference does (its unseeded NaN-climate fill draws in (phase, tile) order); any other tensor is the condition
    vector itself, for every tile."""
    if tile_size is None:
        raise ValueError("sample_base_consistency samples in tiles: tile_size is required")
    B, C, H, W = shape
    cond_inputs, grid = _base_tiles(cond_inputs, H, W, tile_size)
    if noise is not None and len(noise) < 1 + (intermediate_t > 0):
        raise ValueError(f"noise has {len(noise)} phases; this call runs {1 + (intermediate_t > 0)}")
    from .stages import trig_mix
    device = model.device
    sigma_data = float(scheduler.config.sigma_data)
    ts = _phase_times(scheduler, intermediate_t, dtype)
    T = tile_size
    window = _window(weight_window_fn, T, device)
    gen_dev = generator.device if generator is not None else device
    if cond_inputs.ndim == 4:
        cimg = cond_inputs.to(device)
    else:
        cv = cond_inputs.to(device).float()
        cv = cv.reshape(1, -1) if cv.ndim == 1 else cv
        fixed = cv.expand(B, *cv.shape[1:])
    sample = None                                           # the previous phase's normalised canvas [B, C, H, W]
    for k, t in enumerate(ts):
        z = (torch.randn(tuple(shape), generator=generator, device=gen_dev, dtype=dtype) if noise is None
             else torch.as_tensor(noise[k]))
        z = z.to(device).float()
        if cond_inputs.ndim == 4:
            tiles = [(i0, j0, _reference_cond_vector(cimg[..., ic:ic + 4, jc:jc + 4], histogram_raw, cond_means,
                                                     cond_stds, noise_level)) for i0, j0, ic, jc in grid]
        else:
            tiles = [(i0, j0, fixed) for i0, j0, _, _ in grid]

        def run_group(chunk):
            zt = _gather(z, chunk, T)
            if sample is None:
                x = zt                                      # s = 0: x_t = sin t sigma_d z, folded into the program
            else:
                x = trig_mix(_gather(sample, chunk, T), zt, math.cos(t), math.sin(t) * sigma_data)
            solve = get_consistency_solve(model, B * len(chunk), T, T, t, sigma_data, from_unit_noise=sample is None)
            return solve.run(x, None, conditional_inputs=[torch.cat([cvec for _, _, cvec in chunk], dim=0)])

        last = k == len(ts) - 1
        sample = _blend_tiles(tiles, tile_batch, B, C, H, W, window, run_group, sigma_data if last else 1.0)
    return sample.to(dtype)


def cond_inputs_from_snr(cond_snr, device, dtype) -> list:
    """The coarse model's float conditions from the per-channel SNR of its conditioning image
    (training/evaluation/sample_coarse.py:7-26): log(tan(atan(snr)) / 8) in `dtype`, one [rows] tensor per channel."""
    snr = torch.as_tensor(cond_snr).to(device=device, dtype=dtype)
    vals = torch.log(torch.tan(torch.atan(snr)) / 8.0)
    return [vals[:, i].contiguous() for i in range(vals.shape[1])]


@torch.no_grad()
def sample_coarse_tiled(model, scheduler, cond_img: torch.Tensor, cond_snr, *, steps: int = 15,
                        tile_size: Optional[int] = None, tile_stride: Optional[int] = None, weight_window_fn=None,
                        generator: Optional[torch.Generator] = None, dtype=torch.float32,
                        tile_batch: Optional[int] = None):
    """The coarse model's sampler (training/evaluation/sample_coarse.py:29-125): a `steps`-step DPM-Solver++ solve per
    tile, conditioned on the noised conditioning image and on the five float conditions of `cond_snr`.

    cond_snr is [1, C_cond]: one SNR per conditioning channel, shared by the batch.  (The reference runs this shape
    at batch 1 only; with more images its [1]-row conditions fail to stack against the [B]-row noise embedding.)
    The conditioning image is noised first, as cos t_c * cond_img + sin t_c * torch.randn_like(cond_img) with
    t_c = atan(cond_snr), from the global generator of cond_img's device; then every tile draws
    torch.randn(tile, generator=generator) * sigma_0 on cond_img's device, in row-major tile order.  tile_size
    defaults to the image width, tile_stride to tile_size.  Each tile's solve is one fused graph; `tile_batch` tiles
    (default: all) are solved together.  Each tile is divided by sigma_d, blended in row-major order and normalised;
    the result is [B, out_channels, H, W] on cond_img's device, in `dtype`.

    Unlike the reference function as shipped, every tile starts from a reset solver: the reference raises IndexError
    on the second tile because its stateful scheduler is never reset (SURVEY.md section 0 item 7), so its only
    working case, one tile, is reproduced and the multi-tile result is the per-tile-reset one."""
    if cond_img.ndim != 4:
        raise ValueError(f"cond_img must be [B, C, H, W]; got shape {tuple(cond_img.shape)}")
    b, c_cond, h, w = cond_img.shape
    cond_snr = torch.as_tensor(cond_snr)
    if cond_snr.ndim != 2 or cond_snr.shape[0] != 1 or cond_snr.shape[1] != c_cond:
        raise ValueError(f"cond_snr must be [1, {c_cond}] (one SNR per conditioning channel, shared by the batch); "
                         f"got shape {tuple(cond_snr.shape)}")
    tile_size = tile_size or w
    tile_stride = tile_stride or tile_size
    if tile_size > h or tile_size > w:
        raise ValueError(f"tile_size {tile_size} is larger than the {h}x{w} image")
    device, src = model.device, cond_img.device
    out_channels = int(model.config.get("out_channels") or model.config["in_channels"])
    T = tile_size
    window = _window(weight_window_fn, T, device)
    cond_inputs = [ci.to(device) for ci in cond_inputs_from_snr(cond_snr, src, dtype)]
    t_cond = torch.atan(cond_snr).view(1, -1, 1, 1).to(src)
    cond_img = torch.cos(t_cond) * cond_img + torch.sin(t_cond) * torch.randn_like(cond_img)
    scheduler.set_timesteps(int(steps))
    sigma0 = scheduler.sigmas[0].to(src)
    # every tile carries its initial noise, drawn in row-major tile order
    tiles = [(i0, j0, (torch.randn((b, out_channels, T, T), device=src, generator=generator) * sigma0).to(device))
             for i0 in tile_starts(h, T, tile_stride) for j0 in tile_starts(w, T, tile_stride)]
    cond_d = cond_img.to(device).float()
    sd = float(scheduler.config.sigma_data)

    def run_group(chunk):
        n = b * len(chunk)
        solve = get_diffusion_solve(model, scheduler, n, T, T, int(steps))
        x = torch.cat([z for _, _, z in chunk], dim=0).float()
        conds = [ci.float().expand(n).contiguous() for ci in cond_inputs]
        return solve.run(x, _gather(cond_d, chunk, T), conditional_inputs=conds) / sd

    return _blend_tiles(tiles, tile_batch, b, out_channels, h, w, window, run_group).to(device=src, dtype=dtype)


@torch.no_grad()
def sample_decoder_consistency_tiled(model, scheduler, cond_img: torch.Tensor, noise: torch.Tensor,
                                     tile_size: Optional[int] = None, tile_stride: Optional[int] = None, *,
                                     intermediate_t=None, weight_window_fn=None):
    """n-step TrigFlow consistency sampling per tile (sample_diffusion_decoder.py:129-211): x_t = cos t*s + sin t*z,
    pred = -model(x_t/sigma_d, t), s' = cos t*x_t - sin t*sigma_d*pred; blend; / sigma_d."""
    b, c, h, w = noise.shape
    device, dtype = noise.device, noise.dtype
    cond_img = cond_img.to(device=device, dtype=dtype)
    if cond_img.shape[-2:] != (h, w):
        cond_img = F.interpolate(cond_img, size=(h, w), mode="nearest")
    tile_size = tile_size or min(h, w)
    tile_stride = tile_stride or tile_size
    window = _window(weight_window_fn, tile_size, device)
    sigma_data = float(scheduler.config.sigma_data)
    ts = [math.atan(float(scheduler.sigmas[0]) / sigma_data)]
    if intermediate_t is not None:
        if torch.is_tensor(intermediate_t):
            ts += [float(v) for v in intermediate_t.flatten()]
        elif isinstance(intermediate_t, (list, tuple)):
            ts += [float(v) for v in intermediate_t]
        else:
            ts.append(float(intermediate_t))
    tiles = [(i0, j0) for i0 in tile_starts(h, tile_size, tile_stride) for j0 in tile_starts(w, tile_size, tile_stride)]
    noise32, cond32 = noise.float(), cond_img.float()

    def run_group(chunk):
        samples = torch.zeros((b, c, tile_size, tile_size), device=device, dtype=torch.float32)
        tile_cond = _gather(cond32, chunk, tile_size)
        z = _gather(noise32, chunk, tile_size) * sigma_data
        for t in ts:
            x_t = math.cos(t) * samples + math.sin(t) * z
            tt = torch.full((b,), t, device=device, dtype=torch.float32)
            pred = -model(torch.cat([x_t / sigma_data, tile_cond], dim=1), tt, [])
            samples = math.cos(t) * x_t - math.sin(t) * sigma_data * pred
        return samples

    return _blend_tiles(tiles, 1, b, c, h, w, window, run_group, sigma_data).to(dtype)


@torch.no_grad()
def sample_decoder_diffusion_sharded(model, scheduler, cond_img: torch.Tensor, noise: torch.Tensor, tile_size: int,
                                     tile_stride: int, *, num_steps: int, tile_batch: int = 1, group=None):
    """Multi-GPU form of sample_decoder_diffusion_tiled for ONE canvas (batch 1): every rank holds the full noise /
    conditioning canvas (they are inputs), solves only its stripe of tile rows, and the overlap strips are exchanged
    with the neighbours (inference/sharded.py).  Returns this rank's owned rows [C, rows, W] and their (lo, hi)."""
    from .sharded import ShardedCanvas
    b, c, h, w = noise.shape
    assert b == 1, "one canvas per call"
    device = noise.device
    canvas = ShardedCanvas(c, h, w, tile_size, tile_stride, device, group=group)
    tiles = canvas.my_tiles()
    noise32, cond32 = noise.float(), cond_img.to(device).float()
    group_n = max(1, int(tile_batch))
    for g0 in range(0, len(tiles), group_n):
        chunk = tiles[g0:g0 + group_n]
        solve = get_diffusion_solve(model, scheduler, len(chunk), tile_size, tile_size, num_steps)
        out = solve.run(_gather(noise32, chunk, tile_size), _gather(cond32, chunk, tile_size))
        for t, (i0, j0) in enumerate(chunk):
            canvas.add_tile(out[t].clone(), i0, j0)
        if g0 + len(chunk) >= canvas.n_boundary_tiles():
            canvas.start_exchange()          # boundary rows are done: their strip travels during the interior solves
    canvas.finalize()
    return canvas.normalized_owned(), (canvas.own_lo, canvas.own_hi)


@torch.no_grad()
def sample_autoencoder_tiled(model, images: torch.Tensor, tile_size: Optional[int] = None,
                             tile_stride: Optional[int] = None, *, cond_img: Optional[torch.Tensor] = None,
                             conditional_inputs=None, use_mode: bool = False, weight_window_fn=None,
                             tile_batch: Optional[int] = None):
    """Tiled reconstruction with an EDMAutoencoder (training/evaluation/sample_autoencoder.py:8-58): per tile
    preencode -> postencode -> decode, blended in row-major order; [B, out_channels, H, W] in images' dtype.

    tile_size defaults to the image width, tile_stride to tile_size.  The tiles of `tile_batch` tiles (default: all)
    go through one preencode and one decode call; with use_mode=False each tile still draws its own
    randn_like(std) in row-major order, as the reference's per-tile postencode does.  tile_size must be a multiple of
    64 (three 2x down-samplings to a multiple of 8) and fit in the image; otherwise ValueError before any device work."""
    conditional_inputs = list(conditional_inputs or [])
    b, _, h, w = images.shape
    T = tile_size or w
    stride = tile_stride or T
    if T % 64 or T > h or T > w:
        raise ValueError(f"tile_size {T} on a {h}x{w} image: the GPU path takes tiles that are multiples of 64 and fit "
                         "in the image")
    if model.config["direct_skips"]:
        raise NotImplementedError("direct_skips is not implemented by the GPU path (no shipped autoencoder uses it)")
    device, dtype = images.device, images.dtype
    enc_in = images if cond_img is None else torch.cat([images, cond_img], dim=1)
    enc_in = enc_in.to(model.device).float()
    window = _window(weight_window_fn, T, model.device)
    out_channels = int(model.config.get("out_channels") or images.shape[1])
    tiles = [(i0, j0) for i0 in tile_starts(h, T, stride) for j0 in tile_starts(w, T, stride)]

    def run_group(chunk):
        k = len(chunk)
        cond = [torch.cat([torch.as_tensor(c).to(model.device)] * k, dim=0) for c in conditional_inputs]
        means, logvars = model.preencode(_gather(enc_in, chunk, T), cond)
        latent = torch.cat([model.postencode(means[q * b:(q + 1) * b], logvars[q * b:(q + 1) * b], use_mode=use_mode)
                            for q in range(k)], dim=0)
        return model.decode(latent)

    return _blend_tiles(tiles, tile_batch, b, out_channels, h, w, window, run_group).to(device=device, dtype=dtype)


def _latent_tile_geometry(lh: int, lw: int, tile_size: int, tile_stride: int) -> list:
    """Tiles of decode_autoencoder_latents_tiled (sample_autoencoder.py:97-117): per tile (i0, j0, li0, lj0, i_off,
    j_off) with the latent window [li0, li0 + ceil(tile/8)) clipped to the latents and the output offset
    i0 - 8 * li0.  ValueError where the reference's slice assignment fails with a shape mismatch (a slice shorter than
    the tile), and where the latent window is not a multiple of 8 (the decoder's kernels)."""
    n_lat = math.ceil(tile_size / 8)
    tiles = []
    for i0 in tile_starts(lh * 8, tile_size, tile_stride):
        for j0 in tile_starts(lw * 8, tile_size, tile_stride):
            li0, lj0 = i0 // 8, j0 // 8
            rows, cols = min(lh, li0 + n_lat) - li0, min(lw, lj0 + n_lat) - lj0
            i_off, j_off = i0 - 8 * li0, j0 - 8 * lj0
            if i0 + tile_size > lh * 8 or j0 + tile_size > lw * 8 or i_off + tile_size > 8 * rows or \
                    j_off + tile_size > 8 * cols:
                raise ValueError(f"tile_size {tile_size}, stride {tile_stride} on {lh}x{lw} latents: the tile at "
                                 f"({i0}, {j0}) does not fit the decoded {8 * rows}x{8 * cols} latent window or the "
                                 f"{lh * 8}x{lw * 8} output")
            if rows % 8 or cols % 8:
                raise ValueError(f"tile_size {tile_size}: latent windows of {rows}x{cols}; the GPU path decodes "
                                 "latent tiles that are multiples of 8")
            tiles.append((i0, j0, li0, lj0, i_off, j_off))
    return tiles


@torch.no_grad()
def decode_autoencoder_latents_tiled(model, latents: torch.Tensor, tile_size: Optional[int] = None,
                                     tile_stride: Optional[int] = None, *, weight_window_fn=None,
                                     tile_batch: Optional[int] = None):
    """Tiled decoding of latents with an EDMAutoencoder (training/evaluation/sample_autoencoder.py:61-119).

    tile_size None decodes the whole tensor in one call.  Otherwise tile_size / tile_stride are in output pixels (8
    per latent): each tile decodes the latents [i0 // 8, i0 // 8 + ceil(tile / 8)), clipped, and keeps the tile_size
    pixels from offset i0 - 8 * (i0 // 8); tiles are blended in row-major order.  The latent windows of `tile_batch`
    tiles (default: all) go through one decode call.  Geometries the reference cannot blend, or whose latent windows
    are not multiples of 8, raise ValueError before any device work."""
    b, _, lh, lw = latents.shape
    if model.config["direct_skips"]:
        raise NotImplementedError("direct_skips is not implemented by the GPU path (no shipped autoencoder uses it)")
    if tile_size is None:
        if lh % 8 or lw % 8:
            raise ValueError(f"{lh}x{lw} latents: the GPU path decodes latents that are multiples of 8")
        return model.decode(latents)
    T = tile_size
    tiles = _latent_tile_geometry(lh, lw, T, tile_stride or T)
    device, dtype = latents.device, latents.dtype
    lat = latents.to(model.device).float()
    window = _window(weight_window_fn, T, model.device)
    out_channels = int(model.config.get("out_channels") or model.config.get("in_channels") or 1)
    n_lat = math.ceil(T / 8)

    def run_group(chunk):
        out = model.decode(torch.cat([lat[..., li0:li0 + n_lat, lj0:lj0 + n_lat] for _, _, li0, lj0, _, _ in chunk]))
        # each tile keeps the T x T pixels at its own offset in its decoded latent window
        return torch.cat([out[q * b:(q + 1) * b, :, io:io + T, jo:jo + T] for q, (*_, io, jo) in enumerate(chunk)])

    out = _blend_tiles(tiles, tile_batch, b, out_channels, lh * 8, lw * 8, window, run_group)
    return out.to(device=device, dtype=dtype)
