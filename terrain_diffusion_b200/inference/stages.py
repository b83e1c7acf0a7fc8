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
                       (tdx_window_to_cond).  `decoder_stage_tiles` solves a batch of decoder windows with a
                       batch-invariant program, so every window is bit-identical to its `decoder_stage_tile`.
  coarse stage         `get_diffusion_solve`: the 20-step DPM-Solver++ solve as one graph, the embeddings of all steps
                       from one batched call.  De-normalisation, the channel-1 difference, `coarse_pooling` and the
                       packed output are one launch (tdx_coarse_epilogue).  `coarse_stage_tiles` solves a batch of
                       windows: its inputs are one launch (tdx_coarse_condition) and its solve is batch-invariant, so
                       every window is bit-identical to its `coarse_stage_tile`.
  latent stage         `latent_stage_tiles`: one consistency phase of a padded batch of 64^2 tiles.  With
                       batch_invariant=True every tile's embedding row is one CTA of tdx_latent_embed and the program is
                       planned at a fixed anchor, so every tile is bit-identical to a one-tile call of itself.

Noise comes from the bit-compatible GPU generator (same seeds as the reference), nothing synchronises with the host and
nothing leaves the GPU.  Taken as arguments: the synthetic conditioning map of the coarse stage (built on the device by
inference/synthetic_map.py, or by a caller's `conditioning_fn`) and the blended dependency windows the canvas engine
hands to each callback.
"""
from __future__ import annotations

import math
import operator

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


DECODER_BATCH_SIZES = (1, 2, 4)          # not 8 or 16: ~2 GB of activations per 512^2 window (DESIGN.md section 5)


@torch.no_grad()
def decoder_stage_tiles(model, seed: int, ctxs, latents_windows, weight_window: torch.Tensor, t_list,
                        tile_size: int = 512, tile_stride: int = 384, sigma_data: float = 0.5,
                        latent_compression: int = 8) -> list:
    """decoder_stage_tile for a batch of windows: ctxs [(0, i, j), ...] with their packed [6, T/lc, T/lc] latent
    windows (a list of CUDA or CPU tensors, or one [n, 6, T/lc, T/lc] tensor).  Returns the packed [2, T, T] windows
    (views of one device tensor), each bit-identical to decoder_stage_tile of its window whatever the rest of the batch
    is: every launch but the consistency program is elementwise, in that function's fp32 order, and the program is
    batch-invariant.  The batch is padded to the next of DECODER_BATCH_SIZES by repeating window 0, so that few
    programs exist per model.  At most DECODER_BATCH_SIZES[-1] windows per call."""
    if len(ctxs) != len(latents_windows):                        # argument errors before any device work
        raise ValueError(f"decoder_stage_tiles: {len(ctxs)} windows but {len(latents_windows)} latent windows")
    top = DECODER_BATCH_SIZES[-1]
    if len(ctxs) > top:
        raise ValueError(f"decoder_stage_tiles: {len(ctxs)} windows, at most {top} per call")
    T, lc = tile_size, latent_compression
    want = (6, T // lc, T // lc)
    if isinstance(latents_windows, torch.Tensor):
        shapes = [tuple(latents_windows.shape[1:])] if latents_windows.dim() == 4 else [tuple(latents_windows.shape)]
    else:
        shapes = [tuple(torch.as_tensor(w).shape) for w in latents_windows]
    bad = [s for s in shapes if s != want]
    if bad:
        raise ValueError(f"decoder_stage_tiles: latent windows must be {list(want)}, got {list(bad[0])}")
    if not ctxs:
        return []
    dev = model.device
    n = len(ctxs)
    if isinstance(latents_windows, torch.Tensor):
        lat = _f32(latents_windows, dev)
    elif all(torch.as_tensor(w).device.type == "cpu" for w in latents_windows):     # host windows: ONE copy
        lat = _f32(torch.stack([torch.as_tensor(w) for w in latents_windows]), dev)
    else:
        lat = torch.stack([_f32(torch.as_tensor(w), dev) for w in latents_windows])
    origins = [(c[1] * tile_stride, c[2] * tile_stride) for c in ctxs]
    m = padded_batch_size(n, top)
    if m > n:      # padding repeats window 0 at the inputs: its condition and its noise
        lat = torch.cat([lat, lat[:1].expand(m - n, -1, -1, -1)], dim=0)
        origins += [origins[0]] * (m - n)
    cond = window_to_cond(lat, 4, lc)
    sample = None
    for k, t in enumerate(t_list):
        t = float(t)
        z = gaussian_noise_patches(seed + 5819 + k, origins, T, T, 1, T, T, device=dev)
        last = k == len(t_list) - 1
        # one window: the program of decoder_stage_tile itself (a batch-invariant plan at one image is that plan)
        solve = get_consistency_solve(model, m, T, T, t, sigma_data, from_unit_noise=(k == 0),
                                      out_scale=1.0 / sigma_data if last else 1.0, batch_invariant=m > 1)
        x = z if k == 0 else trig_mix(sample, z, math.cos(t), math.sin(t) * sigma_data)
        sample = solve.run(x, cond)
    return list(pack_weighted(sample[:n], _f32(weight_window, dev)))


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


LATENT_BATCH_SIZES = (1, 2, 4, 8, 16)
LATENT_EMBED_MAX_CHANNELS = 1024         # tdx_latent_embed: one CTA per row, the row's embedding in registers


def latent_embed_spec(model) -> dict:
    """What tdx_latent_embed needs to know of the base model, read from its config: a positional noise embedding (its
    dims a multiple of 4, at most 512), exactly one `tensor` conditional input of 52 + n_tail values and at most 1024
    embedding channels, and the mp_sum weights of the two embeddings in fp32 as _host_embedding uses them.  Any other
    embedding configuration raises ValueError."""
    cfg = dict(model.config)
    conds = [list(c) for c in (cfg.get("conditional_inputs") or [])]
    mults = cfg.get("model_channel_mults") or [1, 2, 3, 4]
    mc = cfg.get("model_channels", 128)
    noise_dims = mc if cfg.get("noise_emb_dims") is None else cfg["noise_emb_dims"]
    emb = cfg.get("emb_channels") or mc * max(mults)
    if (cfg.get("fourier_scale") != "pos" or not 4 <= noise_dims <= 512 or noise_dims % 4 or len(conds) != 1
            or conds[0][0] != "tensor" or not 53 <= int(conds[0][1]) <= 128 or emb > LATENT_EMBED_MAX_CHANNELS):
        raise ValueError("the batch-invariant latent stage embeds on the device and supports a positional noise "
                         "embedding (a multiple of 4 dims, at most 512), one 'tensor' conditional input of 53..128 "
                         f"values and at most {LATENT_EMBED_MAX_CHANNELS} embedding channels; this model has "
                         f"fourier_scale={cfg.get('fourier_scale')!r}, noise_emb_dims={noise_dims}, "
                         f"conditional_inputs={conds}, emb_channels={emb}")
    w32 = torch.tensor([1.0, float(conds[0][2])], dtype=torch.float32)   # _host_embedding's mp_sum weights and norm
    return dict(noise_dims=int(noise_dims), emb_channels=int(emb), cond_dims=int(conds[0][1]), w_noise=float(w32[0]),
                w_cond=float(w32[1]), w_norm=float(torch.linalg.vector_norm(w32)))


def latent_plan_images(top: int) -> int:
    """The image count the batch-invariant latent programs plan their launches at (the anchor): the largest padded
    batch, so that a full batch runs its free plan (DESIGN.md section 5 gives the measurement behind the choice)."""
    return int(top)


def latent_embedding(model, coarse: torch.Tensor, histogram_raw, cond_means, cond_stds, t: float, out: torch.Tensor,
                     cond_vec: torch.Tensor | None = None) -> torch.Tensor:
    """The base model's embedding rows of n latent tiles in one launch (tdx_latent_embed): coarse [n, 7, 4, 4] packed
    coarse windows (contiguous fp32 on the model's device) -> out [n, E], row r a function of coarse[r] alone.  What
    latent_stage_tiles + process_latent_conditioning + EDMUnet2D._host_embedding compute, at noise level 0 and label t,
    in one fixed fp32 order per row.  histogram_raw: [H] or [1, H], shared by every row.  cond_vec [n, 52 + H + 1]
    receives the conditioning vectors when given."""
    spec = latent_embed_spec(model)
    fw = model.folded()
    dev = coarse.device
    n = coarse.shape[0]
    hist = torch.as_tensor(histogram_raw, dtype=torch.float32).cpu().reshape(-1)
    level = ((torch.tensor(0.0, dtype=torch.float32) - 0.5) * math.sqrt(12)).reshape(1)   # process_latent_conditioning's
    tail = _const_on(dev, torch.cat([hist, level]))
    dims = [16, 16, 4, 16, hist.numel(), 1]
    if sum(dims) != spec["cond_dims"]:
        raise ValueError(f"latent_embedding: {hist.numel()} histogram values make a {sum(dims)}-value conditioning "
                         f"vector; the model takes {spec['cond_dims']}")
    E = spec["emb_channels"]
    for name, ten, shape in (("coarse", coarse, (n, 7, 4, 4)), ("out", out, (n, E)),
                             ("cond_vec", cond_vec, (n, sum(dims)))):
        if ten is not None and (tuple(ten.shape) != shape or ten.dtype != torch.float32 or not ten.is_contiguous()
                                or ten.device != fw.device):
            raise ValueError(f"latent_embedding: {name} must be a contiguous fp32 {list(shape)} tensor on "
                             f"{fw.device}, got {ten.dtype} {tuple(ten.shape)} on {ten.device}")
    g = fw.g
    L.call(L.lib().tdx_latent_embed, dev, out.data_ptr(), None if cond_vec is None else cond_vec.data_ptr(),
           coarse.data_ptr(), _const_on(dev, cond_means).data_ptr(), _const_on(dev, cond_stds).data_ptr(),
           tail.data_ptr(), tail.numel(), _concat_scales(dims, dev).data_ptr(), g["noise_freqs"].data_ptr(),
           g["noise_linear"].data_ptr(), g["cond0"].data_ptr(), spec["noise_dims"], E, float(t), spec["w_noise"],
           spec["w_cond"], spec["w_norm"], n)
    return out


def _check_latent_arguments(model, ctxs, samples, cond_imgs, histogram_raw, top: int) -> None:
    """The batch-invariant latent stage's argument errors, raised before any device work."""
    n = len(ctxs)
    if len(cond_imgs) != n:
        raise ValueError(f"latent_stage_tiles: {n} tiles but {len(cond_imgs)} coarse windows")
    if samples is not None and len(samples) != n:
        raise ValueError(f"latent_stage_tiles: {n} tiles but {len(samples)} samples")
    if n > top:
        raise ValueError(f"latent_stage_tiles: {n} tiles, at most {top} per batch-invariant call")
    bad = [tuple(torch.as_tensor(c).shape) for c in cond_imgs if tuple(torch.as_tensor(c).shape) != (7, 4, 4)]
    if bad:
        raise ValueError(f"latent_stage_tiles: coarse windows must be [7, 4, 4], got {list(bad[0])}")
    shapes = [tuple(torch.as_tensor(s).shape) for s in (samples or []) if s is not None]
    bad = [sh for sh in shapes if sh != (6, LATENT_TILE, LATENT_TILE)]
    if bad:
        raise ValueError(f"latent_stage_tiles: samples must be [6, {LATENT_TILE}, {LATENT_TILE}], got {list(bad[0])}")
    if 0 < len(shapes) < n:
        raise ValueError("latent_stage_tiles: samples must be all None (first phase) or all windows")
    hist = torch.as_tensor(histogram_raw)
    if hist.dim() > 2 or (hist.dim() == 2 and hist.shape[0] != 1):
        raise ValueError(f"latent_stage_tiles: the batch-invariant stage takes one shared histogram ([H] or [1, H]), "
                         f"got {list(hist.shape)}")
    latent_embed_spec(model)


@torch.no_grad()
def latent_stage_tiles(model, seed: int, ctxs, samples, cond_imgs, t: float, weight_window: torch.Tensor,
                       histogram_raw, cond_means, cond_stds, seed_offset: int = 0, sigma_data: float = 0.5,
                       pad_batch_to=None, batch_invariant: bool = False) -> list:
    """One consistency phase of the latent stage for a batch of window indices (world_pipeline.py:1052-1131).
    samples: None (first phase) or packed [6, 64, 64] windows of the previous phase's canvas; cond_imgs: packed
    [7, 4, 4] coarse windows.  Returns the packed [6, 64, 64] tiles (views of one device tensor).
    batch_invariant: every tile comes out bit-identical to a one-tile call of itself, whatever else is in the batch.
    Its embedding rows are computed on the device per tile (latent_embedding) and the program is planned at the
    anchor latent_plan_images(top), top = pad_batch_to or 16, at every padded batch size; so a tile's bits depend on
    top (the pipeline's largest latents_batch_size) and at most top tiles are taken per call."""
    if batch_invariant:
        top = int(pad_batch_to or LATENT_BATCH_SIZES[-1])
        _check_latent_arguments(model, ctxs, samples, cond_imgs, histogram_raw, top)
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
    if not batch_invariant:
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
    if batch_invariant:
        m = padded_batch_size(n, top)
        if m > n:  # padding repeats tile 0 at the inputs; the anchored program keeps the real tiles' bits
            x = torch.cat([x, x[:1].expand(m - n, -1, -1, -1)], dim=0)
            coarse = torch.cat([coarse, coarse[:1].expand(m - n, -1, -1, -1)], dim=0)
        solve = get_consistency_solve(model, m, T, T, t, sigma_data, from_unit_noise=first, out_scale=1.0 / sigma_data,
                                      batch_invariant=True, plan_images=latent_plan_images(top))
        latent_embedding(model, coarse.contiguous(), histogram_raw, cond_means, cond_stds, t, solve.emb_all)
        sample = solve.run(x, None, embedding_ready=True)
        return list(pack_weighted(sample[:n], _f32(weight_window, dev)))
    m = padded_batch_size(n, pad_batch_to) if pad_batch_to else n
    if m > n:   # the reference pads to {1,2,4,8,16} under torch.compile (:393-398, 1107-1118): one plan per size
        x = torch.cat([x, x[:1].expand(m - n, -1, -1, -1)], dim=0)
        cvec = torch.cat([cvec, cvec[:1].expand(m - n, -1)], dim=0)
    solve = get_consistency_solve(model, m, T, T, t, sigma_data, from_unit_noise=first, out_scale=1.0 / sigma_data)
    sample = solve.run(x, None, conditional_inputs=[cvec])
    return list(pack_weighted(sample[:n], _f32(weight_window, dev)))


# ------------------------------------------------------------------------------------------------ coarse stage
COARSE_POOL_SIZES = tuple(n for n in range(1, COARSE_TILE + 1) if COARSE_TILE % n == 0 and COARSE_STRIDE % n == 0)
_POOL_MODE_FLAGS = {"max": 1, "min": 2}       # tdx_coarse_epilogue's flags; any other mode averages (:994-1002)


def coarse_geometry(pool_size) -> tuple:
    """(tile, stride) of the coarse canvas in pooled cells for `coarse_pooling = pool_size` (world_pipeline.py:961-992):
    window (0, i, j) is still the 64^2 solve at conditioning cells (48 i, 48 j), pooled to tile^2 cells, blended with
    `linear_weight_window(tile)` at a stride of 48 / pool_size.  Raises ValueError unless pool_size is an integer that
    divides both 64 and 48, i.e. one of COARSE_POOL_SIZES."""
    try:
        n = operator.index(pool_size)
    except TypeError:
        n = None
    if n not in COARSE_POOL_SIZES:
        raise ValueError(f"coarse_pooling must be an integer dividing both the coarse tile ({COARSE_TILE}) and its "
                         f"stride ({COARSE_STRIDE}), one of {list(COARSE_POOL_SIZES)}; got {pool_size!r}")
    return COARSE_TILE // n, COARSE_STRIDE // n


def pool_mode_flag(mode) -> int:
    """The reference's `_pool_channel` mode string as tdx_coarse_epilogue's flag: 'max' 1, 'min' 2, anything else avg 0."""
    return _POOL_MODE_FLAGS.get(mode, 0) if isinstance(mode, str) else 0


def coarse_epilogue(sample: torch.Tensor, means: torch.Tensor, stds: torch.Tensor, window: torch.Tensor,
                    pool_size: int = 1, elev_pool_mode: str = "avg", p5_pool_mode: str = "avg",
                    sigma_data: float = 0.5) -> torch.Tensor:
    """[n, 6, 64, 64] raw solve output -> [n, 7, 64/p, 64/p] packed coarse tiles in one launch (world_pipeline.py:948-958):
    de-normalise (x / sigma_data * stds + means), channel 1 = ch0 - ch1, pool by p (channel 0 by elev_pool_mode, 1 by
    p5_pool_mode, 2-5 avg; p = 1 does not pool), cat([v w, w]); bit for bit with the reference's fp32 CPU ops.
    means / stds: 6 fp32 values and window: the [64/p, 64/p] blend weights, all on sample's device."""
    tile, _ = coarse_geometry(pool_size)
    n, c, h, w = sample.shape
    if (c, h, w) != (6, COARSE_TILE, COARSE_TILE) or sample.dtype != torch.float32 or not sample.is_contiguous():
        raise ValueError(f"coarse_epilogue: sample must be a contiguous fp32 [n, 6, 64, 64] tensor, got "
                         f"{sample.dtype} {tuple(sample.shape)}")
    for name, t, shape in (("means", means, (6,)), ("stds", stds, (6,)), ("window", window, (tile, tile))):
        if tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous() or t.device != sample.device:
            raise ValueError(f"coarse_epilogue: {name} must be a contiguous fp32 {list(shape)} tensor on "
                             f"{sample.device}, got {t.dtype} {tuple(t.shape)} on {t.device}")
    out = torch.empty((n, 7, tile, tile), dtype=torch.float32, device=sample.device)
    L.call(L.lib().tdx_coarse_epilogue, sample.device, out.data_ptr(), sample.data_ptr(), means.data_ptr(),
           stds.data_ptr(), window.data_ptr(), n, COARSE_TILE, operator.index(pool_size), pool_mode_flag(elev_pool_mode),
           pool_mode_flag(p5_pool_mode), float(sigma_data))
    return out


@torch.no_grad()
def coarse_stage_tile(model, scheduler, seed: int, ctx, synthetic_map: torch.Tensor, t_cond: torch.Tensor,
                      cond_inputs, weight_window: torch.Tensor, coarse_means, coarse_stds, num_steps: int = 20,
                      pool_size: int = 1, elev_pool_mode: str = "avg", p5_pool_mode: str = "avg") -> torch.Tensor:
    """Coarse window (0, i, j): 20-step DPM-Solver++ solve conditioned on the noised synthetic map
    (world_pipeline.py:909-959).  synthetic_map: the raw [5, 64, 64] conditioning of conditioning cells
    (48 i .. 48 i + 64, 48 j .. 48 j + 64) whatever the pooling, a CUDA or CPU tensor (the pipeline's device synthesis,
    inference/synthetic_map.py, or its `conditioning_fn`).  Returns the packed [7, 64/p, 64/p] tile, p = pool_size (see coarse_geometry / coarse_epilogue);
    weight_window is the [64/p, 64/p] blend window."""
    coarse_geometry(pool_size)                                   # argument errors before any device work
    dev = model.device
    T = COARSE_TILE
    y0, x0 = ctx[1] * COARSE_STRIDE, ctx[2] * COARSE_STRIDE      # = i * (48 // p) * p: p divides 48 (:919-920)
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
    return coarse_epilogue(sample.contiguous(), means, stds, _f32(weight_window, dev), pool_size, elev_pool_mode,
                           p5_pool_mode, float(scheduler.config.sigma_data))[0]


def coarse_condition(maps: torch.Tensor, cond_noise: torch.Tensor, sample_noise: torch.Tensor, means: torch.Tensor,
                     stds: torch.Tensor, t_cond: torch.Tensor, sigma0: float) -> tuple:
    """The solve inputs of n coarse windows in one launch (world_pipeline.py:921-933), bit for bit with
    coarse_stage_tile's torch ops: cond = cos(t) * ((map - mean) / std) + sin(t) * cond_noise over the five map channels
    and sample = sample_noise * sigma0.  maps, cond_noise [n, 5, 64, 64] and sample_noise [n, 6, 64, 64] fp32 on one
    device; means / stds: the 6 model statistics (the map's channels use 0, 2, 3, 4, 5); t_cond: the 5 noise angles.
    Returns (cond, sample)."""
    n = maps.shape[0]
    dev = maps.device
    shapes = ((maps, (n, 5, COARSE_TILE, COARSE_TILE)), (cond_noise, (n, 5, COARSE_TILE, COARSE_TILE)),
              (sample_noise, (n, 6, COARSE_TILE, COARSE_TILE)))
    for t, shape in shapes:
        if tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous() or t.device != dev:
            raise ValueError(f"coarse_condition: expected a contiguous fp32 {list(shape)} tensor on {dev}, got "
                             f"{t.dtype} {tuple(t.shape)} on {t.device}")
    sel = [0, 2, 3, 4, 5]                                        # model statistics of the map's five channels (:925)
    m5, s5 = means[sel].contiguous(), stds[sel].contiguous()
    tc = _const_on(dev, t_cond).view(-1)
    cos_t, sin_t = torch.cos(tc), torch.sin(tc)                  # the same device ops as coarse_stage_tile's
    cond = torch.empty_like(maps)
    sample = torch.empty_like(sample_noise)
    L.call(L.lib().tdx_coarse_condition, dev, cond.data_ptr(), sample.data_ptr(), maps.data_ptr(),
           cond_noise.data_ptr(), sample_noise.data_ptr(), m5.data_ptr(), s5.data_ptr(), cos_t.data_ptr(),
           sin_t.data_ptr(), float(sigma0), n, COARSE_TILE * COARSE_TILE)
    return cond, sample


COARSE_BATCH_SIZES = (1, 2, 4, 8, 16)


@torch.no_grad()
def coarse_stage_tiles(model, scheduler, seed: int, ctxs, synthetic_maps, t_cond: torch.Tensor, cond_inputs,
                       weight_window: torch.Tensor, coarse_means, coarse_stds, num_steps: int = 20, pool_size: int = 1,
                       elev_pool_mode: str = "avg", p5_pool_mode: str = "avg") -> list:
    """coarse_stage_tile for a batch of windows: ctxs [(0, i, j), ...] with their raw [5, 64, 64] conditioning maps
    (a list of CUDA or CPU tensors, or one [n, 5, 64, 64] tensor).  Returns the packed [7, 64/p, 64/p] tiles (views of
    one device tensor), each bit-identical to coarse_stage_tile of its window whatever the rest of the batch is.  The
    batch is padded to the next of COARSE_BATCH_SIZES, so that at
    most five solve programs exist per model.  At most 16 windows per call."""
    coarse_geometry(pool_size)                                   # argument errors before any device work
    if len(ctxs) != len(synthetic_maps):
        raise ValueError(f"coarse_stage_tiles: {len(ctxs)} windows but {len(synthetic_maps)} conditioning maps")
    if not ctxs:
        return []
    top = COARSE_BATCH_SIZES[-1]
    if len(ctxs) > top:
        raise ValueError(f"coarse_stage_tiles: {len(ctxs)} windows, at most {top} per call")
    dev = model.device
    n, T = len(ctxs), COARSE_TILE
    means = _const_on(dev, torch.as_tensor(coarse_means, dtype=torch.float32))
    stds = _const_on(dev, torch.as_tensor(coarse_stds, dtype=torch.float32))
    if isinstance(synthetic_maps, torch.Tensor):
        maps = _f32(synthetic_maps, dev)
    elif all(torch.as_tensor(m).device.type == "cpu" for m in synthetic_maps):   # host maps: ONE copy
        maps = _f32(torch.stack([torch.as_tensor(m) for m in synthetic_maps]), dev)
    else:
        maps = torch.stack([_f32(torch.as_tensor(m), dev) for m in synthetic_maps])
    origins = [(c[1] * COARSE_STRIDE, c[2] * COARSE_STRIDE) for c in ctxs]
    cond_noise = gaussian_noise_patches(seed, origins, T, T, 5, T, T, device=dev)
    sample_noise = gaussian_noise_patches(seed + 1, origins, T, T, 6, T, T, device=dev)
    m = padded_batch_size(n, top)
    solve = get_diffusion_solve(model, scheduler, m, T, T, num_steps, batch_invariant=True)
    cond, sample = coarse_condition(maps, cond_noise, sample_noise, means, stds, t_cond, float(scheduler.sigmas[0]))
    if m > n:      # padding repeats window 0; a batch-invariant solve keeps the real windows' bits
        cond = torch.cat([cond, cond[:1].expand(m - n, -1, -1, -1)], dim=0)
        sample = torch.cat([sample, sample[:1].expand(m - n, -1, -1, -1)], dim=0)
    out = solve.run(sample, cond, conditional_inputs=[_const_on(dev, c) for c in cond_inputs])
    return list(coarse_epilogue(out[:n].contiguous(), means, stds, _f32(weight_window, dev), pool_size, elev_pool_mode,
                                p5_pool_mode, float(scheduler.config.sigma_data)))
