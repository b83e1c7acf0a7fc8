"""The terrain decode of the generative evaluations on the device.

Every evaluation driver of the reference (evaluation/base_consistency.py, base_diffusion.py and the
infinite_consistency*.py drivers) ends in `_decode_latents_to_terrain` (base_consistency.py:34-72): base-model samples
[B, 5, h, w] (four latent channels, then the low-frequency elevation) become [B, 1, 8h, 8w] terrain in signed-sqrt
metres, through a consistency decode of the residual and the Laplacian read-out.  `decode_latents_to_terrain` takes
the same positional arguments, so a driver only swaps its import, and runs

  * the decode as one fused consistency program (get_consistency_solve) per phase for each group of images, the
    later phases mixed in by tdx_trig_mix (stages.trig_mix), blended and divided by sigma_data on a BlendCanvas;
  * the read-out (de-normalisation, laplacian_denoise, laplacian_decode) as ONE batched call, tdx_eval_terrain,
    bit-identical per image to the single-plane chain of inference/postproc.py.

Nothing is copied to the host between the samples and the terrain.  `normalize_uint8_three_channel` is the drivers'
`_normalize_uint8_three_channel`, as torch ops on the samples' device.

The decoder evaluations (evaluation/decoder_consistency.py and tiled_decoder_consistency.py) measure the decoder
itself on the dataset's residuals: `decoder_eval_terrain` is one batch of their loop, the tiled two-step TrigFlow decode
as one fused program per step and the read-out of the generated and the real residual against the pre-padded
low-frequency plane as one `padded_terrain` call (tdx_eval_padded_terrain).
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from .. import _lib as L
from .postproc import LOWFREQ_MEAN, LOWFREQ_STD
from .samplers import _blend_tiles, _gather, _window, get_consistency_solve
from .stages import trig_mix
from .tiling import tile_starts

DATASET_ATTRS = ("latents_mean", "latents_std", "residual_mean", "residual_std")


def _phase_times(scheduler, inter_t) -> list:
    """The consistency times as sample_decoder_consistency_tiled forms them (sample_diffusion_decoder.py:171-187): the
    fp32 atan(sigma_0 / sigma_d), then every entry of `inter_t` (None: none) rounded to fp32."""
    sigma_data = float(scheduler.config.sigma_data)
    s0 = float(scheduler.sigmas[0])
    ts = [torch.atan(torch.as_tensor(s0 / sigma_data, dtype=torch.float32))]
    if inter_t is not None:
        if torch.is_tensor(inter_t):
            ts += [v.to(torch.float32) for v in inter_t.detach().cpu().flatten()]
        elif isinstance(inter_t, (list, tuple)):
            ts += [torch.tensor(float(v), dtype=torch.float32) for v in inter_t]
        else:
            ts.append(torch.tensor(float(inter_t), dtype=torch.float32))
    return [float(t) for t in ts]


def _stats(val_dataset) -> tuple:
    """(latents_mean, latents_std, residual_mean, residual_std) of `val_dataset` (or its `.base_dataset`)."""
    base = val_dataset.base_dataset if hasattr(val_dataset, "base_dataset") else val_dataset
    missing = [a for a in DATASET_ATTRS if not hasattr(base, a)]
    if missing:
        raise AttributeError(f"decode_latents_to_terrain: the dataset has no {', '.join(missing)} (it needs "
                             f"{', '.join(DATASET_ATTRS)}, on itself or on its .base_dataset)")
    return tuple(getattr(base, a) for a in DATASET_ATTRS)


def _scalar(v, name: str, fn: str = "decode_latents_to_terrain") -> float:
    t = torch.as_tensor(v)
    if t.numel() != 1:
        raise ValueError(f"{fn}: {name} must be a scalar, got shape {tuple(t.shape)}")
    return float(t.reshape(()))


def eval_terrain(residual: torch.Tensor, lowfreq: torch.Tensor, residual_mean: float, residual_std: float,
                 denoise: bool = True, signed_square: bool = False) -> torch.Tensor:
    """The batched read-out (tdx_eval_terrain): residual [B, H, W] and lowfreq [B, h, w], CUDA fp32 in normalised units
    (H = 8h, W = 8w) -> terrain [B, H, W]: laplacian_decode(laplacian_denoise(...)) of the de-normalised planes, as
    `_decode_latents_to_terrain` composes them, optionally followed by sign(x) x^2."""
    ok = all(isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 3
             for t in (residual, lowfreq))
    if not ok or residual.device != lowfreq.device:
        raise L.TdxError("eval_terrain: residual and lowfreq must be CUDA float32 [B, H, W] / [B, h, w] tensors on one "
                         "device (the read-out has no CPU path)")
    b, h, w = lowfreq.shape
    if tuple(residual.shape) != (b, 8 * h, 8 * w):
        raise ValueError(f"eval_terrain: residual is {tuple(residual.shape)}; lowfreq {tuple(lowfreq.shape)} needs "
                         f"{(b, 8 * h, 8 * w)}")
    residual, lowfreq = residual.contiguous(), lowfreq.contiguous()
    H, W = 8 * h, 8 * w
    out = torch.empty((b, H, W), dtype=torch.float32, device=residual.device)
    n_scratch = 2 * b * (H + 16) * (W + 16)
    scratch = torch.empty((n_scratch,), dtype=torch.float32, device=residual.device)
    L.call(L.lib().tdx_eval_terrain, out.device, residual.data_ptr(), lowfreq.data_ptr(), b, h, w, float(residual_mean),
           float(residual_std), LOWFREQ_MEAN, LOWFREQ_STD, int(bool(denoise)), int(bool(signed_square)), out.data_ptr(),
           scratch.data_ptr(), n_scratch)
    return out


@torch.no_grad()
def decode_latents_to_terrain(samples: torch.Tensor, val_dataset, decoder_model, scheduler, generator, inter_t,
                              disable_laplacian_denoising: bool = False, *, noise: Optional[torch.Tensor] = None,
                              signed_square: bool = False, decoder_batch_size: Optional[int] = None) -> torch.Tensor:
    """`_decode_latents_to_terrain` (evaluation/base_consistency.py:34-72) on the device: samples [B, 5, h, w] ->
    terrain CUDA fp32 [B, 1, 8h, 8w].

    The latents are normalised (latents / latents_std + latents_mean) and nearest-upsampled x8; one
    torch.randn((B, 1, 8h, 8w), generator=generator) is drawn on the samples' device in their dtype, as the reference
    draws it (or `noise` is used instead, and the generator is not touched).  The residual is decoded as
    sample_decoder_consistency_tiled(tile_size=8h, tile_stride=8h, intermediate_t=inter_t) does it: tiles of 8h x 8h
    (one per image when the image is square), one TrigFlow step at atan(sigma_0 / sigma_d) and one at each entry of
    inter_t, the same z in every phase, blended in row-major order and divided by sigma_d.  Each group of
    `decoder_batch_size` images (default: all) runs one fused program per phase.  Then the residual is de-normalised
    (x * residual_std + residual_mean), the low-frequency plane too (x * 38.6 - 31.4), laplacian_denoise(sigma=5)
    runs unless disable_laplacian_denoising, and laplacian_decode(extrapolate=True) gives the terrain; signed_square
    applies sign(x) x^2 on top (metres instead of signed-sqrt metres).

    ValueError / AttributeError / TdxError before any device work for samples that are not a CUDA float
    [B, 5, h, w] tensor with h, w multiples of 8 and w >= h (the reference's square tiles of 8h must fit the width),
    a dataset without latents_mean, latents_std, residual_mean and residual_std, or a `noise` of the wrong shape."""
    if not isinstance(samples, torch.Tensor) or samples.dim() != 4 or samples.shape[1] != 5:
        raise ValueError(f"decode_latents_to_terrain: samples must be [B, 5, h, w] (4 latent channels, then the "
                         f"low-frequency elevation); got {tuple(getattr(samples, 'shape', ()))}")
    B, _, h, w = samples.shape
    if B < 1 or h < 8 or w < 8 or h % 8 or w % 8:
        raise ValueError(f"decode_latents_to_terrain: {h}x{w} latents (batch {B}); the decoder takes latents whose "
                         "sides are non-zero multiples of 8 (images of multiples of 64 pixels)")
    if w < h:
        raise ValueError(f"decode_latents_to_terrain: {h}x{w} latents; the reference decodes in square tiles of the "
                         "image height, which must fit the width")
    latents_mean, latents_std, residual_mean, residual_std = _stats(val_dataset)
    residual_mean, residual_std = _scalar(residual_mean, "residual_mean"), _scalar(residual_std, "residual_std")
    if not samples.is_cuda or not samples.is_floating_point():
        raise L.TdxError(f"decode_latents_to_terrain: samples must be a CUDA floating-point tensor (there is no CPU "
                         f"path); got {samples.device} {samples.dtype}")
    H, W = 8 * h, 8 * w
    device, dtype = samples.device, samples.dtype
    if noise is not None and (tuple(noise.shape) != (B, 1, H, W) or not noise.is_cuda):
        raise ValueError(f"decode_latents_to_terrain: noise must be a CUDA [B, 1, {H}, {W}] tensor; got "
                         f"{noise.device} {tuple(noise.shape)}")
    group = B if decoder_batch_size is None else int(decoder_batch_size)
    if group < 1:
        raise ValueError(f"decode_latents_to_terrain: decoder_batch_size must be >= 1, got {decoder_batch_size}")

    latents = samples[:, :4]
    lowfreq = samples[:, 4]
    latents = latents / torch.as_tensor(latents_std).to(device) + torch.as_tensor(latents_mean).to(device)
    cond = F.interpolate(latents, size=(H, W), mode="nearest").float()
    if noise is None:
        noise = torch.randn((B, 1, H, W), generator=generator, device=device, dtype=dtype)
    z = noise.to(device).float()

    sigma_data = float(scheduler.config.sigma_data)
    ts = _phase_times(scheduler, inter_t)
    T = H
    window = _window(None, T, device)
    tiles = [(i0, j0) for i0 in tile_starts(H, T, T) for j0 in tile_starts(W, T, T)]
    residual = torch.empty((B, H, W), dtype=torch.float32, device=device)
    for g0 in range(0, B, group):
        g1 = min(B, g0 + group)
        zg, cg = z[g0:g1], cond[g0:g1]

        def run_group(chunk, zg=zg, cg=cg):
            zt, ct = _gather(zg, chunk, T), _gather(cg, chunk, T)
            sample = None
            for k, t in enumerate(ts):
                x = zt if k == 0 else trig_mix(sample, zt, math.cos(t), math.sin(t) * sigma_data)
                solve = get_consistency_solve(decoder_model, zt.shape[0], T, T, t, sigma_data, from_unit_noise=k == 0)
                sample = solve.run(x, ct)
            return sample

        residual[g0:g1] = _blend_tiles(tiles, None, g1 - g0, 1, H, W, window, run_group, sigma_data)[:, 0]
    denoise = not disable_laplacian_denoising
    terrain = eval_terrain(residual, lowfreq.float().contiguous(), residual_mean, residual_std, denoise, signed_square)
    return terrain[:, None]


def padded_terrain(residual: torch.Tensor, lowfreq_padded: torch.Tensor, residual_mean: float, residual_std: float,
                   signed_square: bool = True, crop: Optional[int] = None) -> torch.Tensor:
    """The decoder evaluations' batched read-out (tdx_eval_padded_terrain): residual [B, H, W] in normalised units and
    the pre-padded low-frequency planes [B, h + 2, w + 2], CUDA fp32, H = 8h, W = 8w -> terrain [B, H, W]:
    laplacian_decode(residual * residual_std + residual_mean, lowfreq_padded, pre_padded=True), optionally followed by
    sign(x) x^2, and reduced to the centre crop x crop when `crop` is given."""
    ok = all(isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 3
             for t in (residual, lowfreq_padded))
    if not ok or residual.device != lowfreq_padded.device:
        raise L.TdxError("padded_terrain: residual and lowfreq_padded must be CUDA float32 [B, H, W] / [B, h+2, w+2] "
                         "tensors on one device (the read-out has no CPU path)")
    b, hp, wp = lowfreq_padded.shape
    h, w = hp - 2, wp - 2
    if h < 1 or w < 1 or tuple(residual.shape) != (b, 8 * h, 8 * w):
        raise ValueError(f"padded_terrain: residual is {tuple(residual.shape)} and lowfreq_padded "
                         f"{tuple(lowfreq_padded.shape)}; the read-out takes [B, 8h, 8w] with [B, h+2, w+2], h, w >= 1")
    H, W = 8 * h, 8 * w
    c = 0 if crop is None else int(crop)
    if crop is not None and not 1 <= c <= min(H, W):
        raise ValueError(f"padded_terrain: crop {crop} of a {H}x{W} plane (1..{min(H, W)})")
    residual, lowfreq_padded = residual.contiguous(), lowfreq_padded.contiguous()
    out = torch.empty((b, c or H, c or W), dtype=torch.float32, device=residual.device)
    n_scratch = b * (h + 2) * (W + 16)
    scratch = torch.empty((n_scratch,), dtype=torch.float32, device=residual.device)
    L.call(L.lib().tdx_eval_padded_terrain, out.device, residual.data_ptr(), lowfreq_padded.data_ptr(), b, h, w,
           float(residual_mean), float(residual_std), int(bool(signed_square)), c, out.data_ptr(), scratch.data_ptr(),
           n_scratch)
    return out


def decoder_eval_times(scheduler, intermediate_sigma: float, sigma_data: float) -> list:
    """The TrigFlow times of the decoder evaluations as the drivers form them (decoder_consistency.py:115-119): numpy's
    atan of the scheduler's sigma_0 / sigma_data (fp32, as the sigma table is), then, when intermediate_sigma > 0, the
    float64 atan(intermediate_sigma / sigma_data); both as the fp32 values the model sees."""
    ts = [torch.as_tensor(np.arctan(torch.as_tensor(scheduler.sigmas[0] / sigma_data).numpy()))]
    if intermediate_sigma > 0:
        ts.append(torch.as_tensor(np.arctan(intermediate_sigma / sigma_data)))
    return [float(t.to(torch.float32)) for t in ts]


@torch.no_grad()
def decoder_eval_terrain(model, scheduler, images: torch.Tensor, lowfreq_padded: torch.Tensor, cond_img: torch.Tensor,
                         generator: Optional[torch.Generator], *, residual_mean, residual_std, sigma_data: float = 0.5,
                         tile_size: int = 512, tile_stride: Optional[int] = None, intermediate_sigma: float = 0.065,
                         crop_size: Optional[int] = None, tile_batch: Optional[int] = None) -> tuple:
    """One batch of the decoder evaluations (evaluation/decoder_consistency.py:131-196 and tiled_decoder_consistency.py:
    135-196) on the device: the dataset's images [B, 1, S, S] (residual * sigma_data), lowfreq_padded [B, 1, S/8 + 2,
    S/8 + 2] and cond_img [B, C, S, S] -> (output_full, images_full), the generated and the real terrain in metres,
    CUDA fp32 [B, 1, S, S], or [B, 1, crop_size, crop_size] for the centre crop.  The drivers' metric then takes
    normalize_uint8_three_channel of each.

    Tiles of tile_size start at k * tile_stride (default tile_size // 2) for k in range((S - T) // stride + 1) on both
    axes.  Every tile runs the drivers' two-step TrigFlow loop, one step at atan(sigma_0 / sigma_data) and one at
    atan(intermediate_sigma / sigma_data) (only the first when intermediate_sigma <= 0), each from a fresh
    torch.randn((B, 1, T, T), generator=generator) drawn on the generator's device (images' device for None) in the
    drivers' order, tiles row-major, then steps; all draws happen before the first solve, and leave the generator
    where the drivers leave it.  Each step of `tile_batch` tiles (default: all) with all B images is one fused
    consistency program.  The tiles are blended with the linear window (_get_weights) in row-major order and divided
    by sigma_data; then the generated and the real residual (images / sigma_data) go through ONE padded_terrain call
    (de-normalisation, pre-padded laplacian_decode, signed square, crop).

    ValueError / TdxError before any device work for images that are not square CUDA [B, 1, S, S] tensors with
    S a multiple of 8, inputs whose shapes disagree, or a crop larger than the image.  A tile geometry that leaves
    pixels uncovered (T > S, stride > T, (S - T) % stride != 0 or T < 2) is a ValueError; the drivers divide 0 by 0
    there and hand NaN to the metric, the only place this function does not do what they do."""
    if not all(isinstance(t, torch.Tensor) and t.dim() == 4 for t in (images, lowfreq_padded, cond_img)):
        raise ValueError("decoder_eval_terrain: images, lowfreq_padded and cond_img must be [B, C, H, W] tensors")
    B, C, S, S2 = images.shape
    if B < 1 or C != 1 or S != S2 or S < 8 or S % 8:
        raise ValueError(f"decoder_eval_terrain: images are {tuple(images.shape)}; the drivers decode square "
                         f"[B, 1, S, S] residuals with S a non-zero multiple of 8")
    if tuple(lowfreq_padded.shape) != (B, 1, S // 8 + 2, S // 8 + 2):
        raise ValueError(f"decoder_eval_terrain: lowfreq_padded is {tuple(lowfreq_padded.shape)}; {S}x{S} images "
                         f"need {(B, 1, S // 8 + 2, S // 8 + 2)}")
    if cond_img.shape[0] != B or tuple(cond_img.shape[-2:]) != (S, S):
        raise ValueError(f"decoder_eval_terrain: cond_img is {tuple(cond_img.shape)}; it must be [{B}, C, {S}, {S}]")
    T = int(tile_size)
    stride = T // 2 if tile_stride is None else int(tile_stride)
    if T < 2 or T > S or stride < 1 or stride > T or (S - T) % stride:
        raise ValueError(f"decoder_eval_terrain: tiles of {T} at stride {stride} leave pixels of the {S}x{S} image "
                         "uncovered (the drivers would divide 0 by 0 there)")
    if crop_size is not None and not 1 <= int(crop_size) <= S:
        raise ValueError(f"decoder_eval_terrain: crop_size {crop_size} of a {S}x{S} image")
    if tile_batch is not None and int(tile_batch) < 1:
        raise ValueError(f"decoder_eval_terrain: tile_batch must be >= 1, got {tile_batch}")
    residual_mean = _scalar(residual_mean, "residual_mean", "decoder_eval_terrain")
    residual_std = _scalar(residual_std, "residual_std", "decoder_eval_terrain")
    device = images.device
    if not images.is_cuda or lowfreq_padded.device != device or cond_img.device != device:
        raise L.TdxError(f"decoder_eval_terrain: images, lowfreq_padded and cond_img must be on one CUDA device (there "
                         f"is no CPU path); got {images.device}, {lowfreq_padded.device}, {cond_img.device}")

    sigma_data = float(sigma_data)
    ts = decoder_eval_times(scheduler, float(intermediate_sigma), sigma_data)
    n_tiles = (S - T) // stride + 1
    tiles = [(i * stride, j * stride, i * n_tiles + j) for i in range(n_tiles) for j in range(n_tiles)]
    gen_dev = generator.device if generator is not None else device
    noise = [[torch.randn((B, C, T, T), generator=generator, device=gen_dev) for _ in ts] for _ in tiles]
    cond = cond_img.float()
    window = _window(None, T, device)

    def run_group(chunk):
        ct = _gather(cond, chunk, T)
        sample = None
        for k, t in enumerate(ts):
            zt = torch.cat([noise[q][k] for _, _, q in chunk], dim=0).to(device)
            x = zt if k == 0 else trig_mix(sample, zt, math.cos(t), math.sin(t) * sigma_data)
            solve = get_consistency_solve(model, zt.shape[0], T, T, t, sigma_data, from_unit_noise=k == 0)
            sample = solve.run(x, ct)
        return sample

    output = _blend_tiles(tiles, tile_batch, B, C, S, S, window, run_group, sigma_data)
    residual = torch.cat([output[:, 0], images[:, 0].float() / sigma_data])
    lowfreq = lowfreq_padded[:, 0].float()
    terrain = padded_terrain(residual, torch.cat([lowfreq, lowfreq]), residual_mean, residual_std, True, crop_size)
    return terrain[:B, None], terrain[B:, None]


def normalize_uint8_three_channel(images: torch.Tensor) -> torch.Tensor:
    """The drivers' `_normalize_uint8_three_channel` (base_consistency.py:25-32): each [1, H, W] image of [B, 1, H, W]
    mapped to uint8 around its mid-range over max(range, 255), repeated to three channels."""
    image_min = torch.amin(images, dim=(1, 2, 3), keepdim=True)
    image_max = torch.amax(images, dim=(1, 2, 3), keepdim=True)
    image_range = torch.maximum(image_max - image_min, torch.tensor(255.0, device=images.device))
    image_mid = (image_min + image_max) / 2
    normalized = torch.clamp(((images - image_mid) / image_range + 0.5) * 255, 0, 255)
    return normalized.repeat(1, 3, 1, 1).to(torch.uint8)
