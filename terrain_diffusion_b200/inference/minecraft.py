"""The Minecraft API's read-out on the device (`mc-api`, terrain_diffusion/inference/minecraft_api.py).

After `get()`, the reference's `GET /terrain` (also `/90`, `/45`, `/22`, `/11`) upsamples a padded native window with
torch's CPU bilinear `F.interpolate`, takes a Sobel slope, adds slope-scaled detail noise (scale > 1, noise > 0), derives
climate variables and classifies every pixel into a Minecraft biome id with ~150 full-frame mask operations, all on the
host.  Here one launch of csrc/tdx_biome.cu (`tdx_minecraft_readout`) does all of it per output pixel and writes the
fp32 planes, the int16 biome ids and/or the wire body.

Noise is injected, like the conditioning map: `noise_fn(cfg, i0, j0, h, w) -> fp32 [h, w]` (numpy array or tensor)
returns the generator of configuration `cfg` (a `NoiseConfig`) at x = j0 + c, y = i0 + r for row r, column c, as the
reference calls `gen_from_coords`.  The reference's seven FastNoiseLite generators have five distinct configurations
(`_TEMP_NOISE` = `_SNOW_NOISE`, `_TEMP_NOISE_FINE` = `_SNOW_NOISE_FINE`), so a request calls the provider once per
configuration it needs: a provider must be a pure function of its arguments.  The default provider builds the
reference's generators with pyfastnoiselite.
"""
from __future__ import annotations

import ctypes as C
import functools
from collections import namedtuple

import numpy as np
import torch

from .. import _lib as L
from . import postproc

NoiseConfig = namedtuple("NoiseConfig", "seed frequency octaves lacunarity gain")

# minecraft_api.py:127-186, in the order of the noise planes the kernel reads
TEMP_COARSE = NoiseConfig(12345, 1.0 / 500.0, 3, 2.0, 0.5)      # _TEMP_NOISE, _SNOW_NOISE
TEMP_FINE = NoiseConfig(54321, 1.0 / 128.0, 2, 2.0, 0.5)        # _TEMP_NOISE_FINE, _SNOW_NOISE_FINE
PRECIP = NoiseConfig(12345, 1.0 / 500.0, 5, 2.0, 0.5)           # _PRECIP_NOISE
ELEV_COARSE = NoiseConfig(99999, 1.0 / 24.0, 3, 2.0, 0.5)       # _ELEV_NOISE_COARSE
ELEV_FINE = NoiseConfig(88888, 1.0 / 6.0, 2, 2.0, 0.6)          # _ELEV_NOISE_FINE
NOISE_CONFIGS = (TEMP_COARSE, TEMP_FINE, PRECIP, ELEV_COARSE, ELEV_FINE)
CLIMATE_NOISE, DETAIL_NOISE = (0, 1, 2), (3, 4)


@functools.lru_cache(maxsize=None)
def _generator(cfg: NoiseConfig):
    try:
        from pyfastnoiselite.pyfastnoiselite import FastNoiseLite, FractalType, NoiseType
    except ImportError:
        raise RuntimeError("no noise source: pass noise_fn=... (FastNoiseLite Perlin noise is not part of this "
                           "package) or install pyfastnoiselite, which the default noise provider uses") from None
    g = FastNoiseLite(seed=cfg.seed)
    g.noise_type = NoiseType.NoiseType_Perlin
    g.frequency = cfg.frequency
    g.fractal_type = FractalType.FractalType_FBm
    g.fractal_octaves = cfg.octaves
    g.fractal_lacunarity = cfg.lacunarity
    g.fractal_gain = cfg.gain
    return g


def fastnoiselite_noise(cfg: NoiseConfig, i0: int, j0: int, h: int, w: int) -> np.ndarray:
    """The default `noise_fn`: the reference's pyfastnoiselite generator of `cfg` at x = j0 + c, y = i0 + r
    (minecraft_api.py:324-331, 388-406).  Raises RuntimeError naming pyfastnoiselite and `noise_fn=` without it."""
    g = _generator(cfg)
    xx, yy = np.meshgrid(np.arange(j0, j0 + w, dtype=np.float32), np.arange(i0, i0 + h, dtype=np.float32))
    return g.gen_from_coords(np.array([xx.ravel(), yy.ravel()], dtype=np.float32)).astype(np.float32).reshape(h, w)


def minecraft_window(i1: int, j1: int, i2: int, j2: int, scale: int):
    """Checks a request's arguments as `terrain_window` does (integers only, scale >= 1, non-empty, at most 65535 rows;
    ValueError) and returns the window the elevation is read from and the crop origin in its (upsampled) version:
    (wi1, wj1, wi2, wj2, oi, oj).  Scale 1 (`_handle_1x`, minecraft_api.py:714-727): the window and its 1-pixel ring,
    crop at (1, 1).  Scale >= 2 (`_get_upsampled`, :272-307): the native window padded by 2 pixels."""
    postproc.terrain_window(i1, j1, i2, j2, scale)
    i1, j1, i2, j2, scale = int(i1), int(j1), int(i2), int(j2), int(scale)
    if scale == 1:
        return i1 - 1, j1 - 1, i2 + 1, j2 + 1, 1, 1
    ni1, nj1 = i1 // scale, j1 // scale
    ni2, nj2 = -(-i2 // scale), -(-j2 // scale)
    return ni1 - 2, nj1 - 2, ni2 + 2, nj2 + 2, 2 * scale + i1 - ni1 * scale, 2 * scale + j1 - nj1 * scale


def _noise_scale(noise) -> float:
    if isinstance(noise, bool) or not isinstance(noise, (int, float, np.integer, np.floating)):
        raise ValueError(f"noise must be a number, got {noise!r}")
    return float(noise)


def noise_planes(noise_fn, i1: int, j1: int, H: int, W: int, which, device) -> torch.Tensor:
    """fp32 [5, H, W] on `device`: planes `which` (indices into NOISE_CONFIGS) from one call of `noise_fn` each, the
    others zero."""
    out = torch.zeros((5, H, W), dtype=torch.float32, device=device)
    for k in which:
        v = torch.as_tensor(noise_fn(NOISE_CONFIGS[k], i1, j1, H, W))
        if tuple(v.shape) != (H, W):
            raise ValueError(f"noise_fn returned shape {tuple(v.shape)} for a {H} x {W} window")
        out[k].copy_(v.to(torch.float32))
    return out


def readout(elev: torch.Tensor, climate, noise: torch.Tensor, scale: int, oi: int, oj: int, H: int, W: int,
            noise_scale: float, pixel_size_m: float, native_resolution: float, centre=None, payload: bool = False):
    """One `tdx_minecraft_readout` launch.  Returns (fp32 [7, H, W] = elev, elev_smooth, 5 climate planes (or [2, H, W]
    without climate), int16 biome [H, W]), or with `payload` the wire body as uint8 [4HW].  The scalars are the
    reference's Python doubles, each rounded to fp32 as torch rounds a Python scalar at every op."""
    elev = postproc.check_plane(elev, "minecraft readout(elev)")
    h, w = elev.shape
    if centre is not None:
        centre = postproc.check_plane(centre, "minecraft readout(centre)")
    if climate is not None:
        climate = postproc.check_plane(climate, "minecraft readout(climate)", (5, H, W) if scale == 1 else (5, h, w),
                                       elev.device)
    noise = noise.contiguous()
    detail = int(scale > 1 and noise_scale > 0)
    scalars = (C.c_float(noise_scale * 100.0), C.c_float(noise_scale * 70.0), C.c_float(pixel_size_m),
               C.c_float(native_resolution), C.c_float(40.0 * pixel_size_m / 90.0))
    head = (elev.data_ptr(), h, w, scale, oi, oj, None if centre is None else centre.data_ptr(),
            None if climate is None else climate.data_ptr(), noise.data_ptr(), H, W, detail, *scalars)
    if payload:
        out = torch.empty((4 * H * W,), dtype=torch.uint8, device=elev.device)
        L.call(L.lib().tdx_minecraft_readout, elev.device, *head, None, None, None, None, out.data_ptr())
        return out
    planes = torch.empty((7 if climate is not None else 2, H, W), dtype=torch.float32, device=elev.device)
    biome = torch.empty((H, W), dtype=torch.int16, device=elev.device)
    L.call(L.lib().tdx_minecraft_readout, elev.device, *head, planes[0].data_ptr(), planes[1].data_ptr(),
           planes[2].data_ptr() if climate is not None else None, biome.data_ptr(), None)
    return planes, biome


def request(get_device, native_resolution: float, i1, j1, i2, j2, scale, noise, noise_fn, payload: bool):
    """A whole `/terrain` read-out on `get_device(i1, j1, i2, j2, with_climate) -> {'elev', 'climate'}` (CUDA tensors):
    the argument checks, the reads the reference's handler makes, the noise planes and one launch.  Returns `readout`'s
    result and (H, W)."""
    wi1, wj1, wi2, wj2, oi, oj = minecraft_window(i1, j1, i2, j2, scale)
    noise_scale = _noise_scale(noise)
    i1, j1, scale = int(i1), int(j1), int(scale)
    H, W = int(i2) - i1, int(j2) - j1
    noise_fn = fastnoiselite_noise if noise_fn is None else noise_fn
    if scale == 1:
        slope = get_device(wi1, wj1, wi2, wj2, False)["elev"]
        native = get_device(i1, j1, i1 + H, j1 + W, True)
        centre, pixel_size_m = native["elev"], native_resolution
    else:
        native = get_device(wi1, wj1, wi2, wj2, True)
        slope, centre, pixel_size_m = native["elev"], None, native_resolution / scale
    climate = native["climate"]
    which = (CLIMATE_NOISE if climate is not None else ()) + (DETAIL_NOISE if scale > 1 and noise_scale > 0 else ())
    planes = noise_planes(noise_fn, i1, j1, H, W, which, slope.device)
    out = readout(slope, climate, planes, scale, oi, oj, H, W, noise_scale, pixel_size_m, native_resolution,
                  centre=centre, payload=payload)
    return out, (H, W)
