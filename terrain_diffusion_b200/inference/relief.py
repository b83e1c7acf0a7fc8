"""Shaded relief map on the device: drop-in for terrain_diffusion.inference.relief_map.get_relief_map
(relief_map.py:64-199), the picture the explorer's default `/api/detail.png` mode, `random_sampler.py`, the figure
scripts and the evaluations' `--save-images` branch render from an elevation window.

The reference copies the elevation to the host and runs scipy's `gaussian_filter` twice, `np.gradient` and a GDAL-style
hillshade per scale, matplotlib's `terrain` colormap and an ocean blend on the CPU.  Here that is four launches of
csrc/tdx_relief.cu (statistics, one Gaussian pass per axis for both scales, one fused shade-and-colour pass).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from .. import _lib as L

# matplotlib's `terrain` colormap (matplotlib/_cm.py `_terrain_data`): six (position, RGB) stops, linearly interpolated
TERRAIN_STOPS = ((0.00, (0.2, 0.2, 0.6)), (0.15, (0.0, 0.6, 1.0)), (0.25, (0.0, 0.8, 0.4)),
                 (0.50, (1.0, 1.0, 0.6)), (0.75, (0.5, 0.36, 0.33)), (1.00, (1.0, 1.0, 1.0)))
LUT_SIZE = 256                       # rcParams['image.lut']
MAX_RADIUS = 96                      # tdx_relief_gaussian's limit on int(4 sigma + 0.5)
ALTITUDE_DEG = 45.0                  # sun elevation (relief_map.py:103)


def terrain_lut() -> np.ndarray:
    """fp64 [256, 3]: the table `LinearSegmentedColormap.from_list("terrain", _terrain_data, 256)` builds, channel by
    channel, with `colors._create_lookup_table` (gamma 1)."""
    pos = np.array([p for p, _ in TERRAIN_STOPS], dtype=np.float64) * (LUT_SIZE - 1)
    xind = (LUT_SIZE - 1) * np.linspace(0, 1, LUT_SIZE)
    ind = np.searchsorted(pos, xind)[1:-1]
    distance = (xind[1:-1] - pos[ind - 1]) / (pos[ind] - pos[ind - 1])
    out = np.empty((LUT_SIZE, 3), dtype=np.float64)
    for c in range(3):
        y = np.array([rgb[c] for _, rgb in TERRAIN_STOPS], dtype=np.float64)
        out[:, c] = np.clip(np.concatenate([[y[0]], distance * (y[ind] - y[ind - 1]) + y[ind - 1], [y[-1]]]), 0.0, 1.0)
    return out


def gaussian_taps(sigma: float) -> np.ndarray:
    """fp64 taps of scipy.ndimage.gaussian_filter1d(truncate=4): radius int(4 sigma + 0.5), exp(-0.5 / sigma^2 * x^2)
    normalised by its sum, as scipy's `_gaussian_kernel1d` computes them.  A sigma <= 1e-15 leaves its axis unfiltered
    in scipy; the single tap 1.0 does the same."""
    sigma = float(sigma)
    if sigma <= 1e-15:
        return np.ones(1)
    radius = int(4.0 * sigma + 0.5)
    x = np.arange(-radius, radius + 1)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return phi / phi.sum()


def nanmedian_fill(x: torch.Tensor) -> float:
    """The value the reference replaces NaN with (relief_map.py:107-109): np.nanmedian of the fp32 values -- for an
    even count the fp32 mean of the two middle values -- or 0.0 when it is not finite (all NaN, or an infinite median)."""
    v = torch.sort(x.reshape(-1)[~torch.isnan(x.reshape(-1))]).values
    n = v.numel()
    if n == 0:
        return 0.0
    m = float(v[n // 2]) if n % 2 else float((v[n // 2 - 1:n // 2] + v[n // 2:n // 2 + 1]) / 2)
    return m if math.isfinite(m) else 0.0


_luts: dict = {}


def _lut_on(device: torch.device) -> torch.Tensor:
    if device not in _luts:
        _luts[device] = torch.from_numpy(terrain_lut().astype(np.float32)).to(device)
    return _luts[device]


def _p(t: torch.Tensor):
    return C.c_void_p(t.data_ptr())


def gaussian_filter(x: torch.Tensor, sigmas, *, nan_fill: float | None = None) -> torch.Tensor:
    """scipy.ndimage.gaussian_filter(x, sigma) (mode 'reflect', truncate 4, fp32 between the axes), bit for bit, for one
    or two sigmas in one pair of launches: CUDA fp32 [H, W] -> [len(sigmas), H, W].  With nan_fill, NaN is read as it."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 2):
        raise L.TdxError("gaussian_filter: expected a CUDA float32 [H, W] tensor")
    sigmas = [float(s) for s in sigmas]
    taps = [gaussian_taps(s) for s in sigmas]
    radius = [len(t) // 2 for t in taps]
    if not 1 <= len(sigmas) <= 2 or max(radius) > MAX_RADIUS:
        raise ValueError(f"gaussian_filter: 1 or 2 sigmas with int(4 sigma + 0.5) <= {MAX_RADIUS}, got {sigmas}")
    x = x.contiguous()
    h, w = x.shape
    w64 = np.ascontiguousarray(np.concatenate(taps), dtype=np.float64)
    r32 = (C.c_int32 * len(radius))(*radius)
    with torch.cuda.device(x.device):
        tmp = torch.empty((len(sigmas), h, w), dtype=torch.float32, device=x.device)
        out = torch.empty_like(tmp)
        L.check(L.lib().tdx_relief_gaussian(_p(x), h, w, int(nan_fill is not None),
                                            0.0 if nan_fill is None else float(nan_fill), len(sigmas),
                                            w64.ctypes.data_as(C.POINTER(C.c_double)), r32, _p(tmp), _p(out),
                                            L.current_stream_ptr()))
    return out


def _check_args(elevation, biome, flow, rgb, sigma_large, sigma_small):
    if biome is not None or flow is not None or rgb is not None:
        raise NotImplementedError("get_relief_map: the biome, river (flow) and rgb overlays are not implemented on the "
                                  "device; pass None")
    shape = tuple(elevation.shape) if hasattr(elevation, "shape") else np.shape(elevation)
    if len(shape) != 2 or shape[0] < 2 or shape[1] < 2:
        raise ValueError(f"get_relief_map: elevation must be (H, W) with H, W >= 2 (np.gradient), got {shape}")
    if shape[0] > 65535:
        raise ValueError(f"get_relief_map: at most 65535 rows, got {shape[0]}")
    for s in (sigma_large, sigma_small):
        if int(4.0 * float(s) + 0.5) > MAX_RADIUS:
            raise ValueError(f"get_relief_map: sigma {s} is too large (int(4 sigma + 0.5) must be <= {MAX_RADIUS})")


def get_relief_map(elevation, climate, biome, flow, *, azimuths=(315.0, 45.0, 135.0, 225.0), flow_threshold=7,
                   sigma_large=6.0, sigma_small=1.2, resolution=90, rgb=None, relief=1.0, vmin=None, vmax=None):
    """GDAL-style shaded relief of an elevation window in metres, as RGB fp32 [H, W, 3] in [0, 1] (NaN where the
    elevation is NaN, except where the NaN fill is below sea level: those pixels are ocean-coloured, as in the reference).

    A numpy array or CPU tensor is computed on the current CUDA device and returned as a numpy array (the reference's
    return value); a CUDA tensor returns a CUDA tensor on its device.  Only `azimuths[0]` is used, `climate` and
    `flow_threshold` are ignored, as in the reference.  `biome`, `flow` and `rgb` must be None.

    The reference replaces NaN by the NaN-median before filtering.  To choose that branch the call reads the NaN count
    back to the host (one 4-byte read, which waits for the elevation); only when it is non-zero are the values sorted
    on the device for the median.  `get()` never produces NaN.
    """
    del climate, flow_threshold
    _check_args(elevation, biome, flow, rgb, sigma_large, sigma_small)
    if not torch.cuda.is_available():
        raise L.TdxError("get_relief_map runs on a CUDA device and none is available (there is no CPU path)")
    on_device = isinstance(elevation, torch.Tensor) and elevation.is_cuda
    if on_device:
        elev = elevation.detach().float()
    else:
        host = elevation.detach().cpu().numpy() if isinstance(elevation, torch.Tensor) else np.asarray(elevation)
        elev = torch.from_numpy(np.ascontiguousarray(host, dtype=np.float32)).cuda()
    with torch.cuda.device(elev.device):
        out = _relief(elev.contiguous(), azimuths, sigma_large, sigma_small, resolution, relief, vmin, vmax)
    return out if on_device else out.cpu().numpy()


def _relief(elev, azimuths, sigma_large, sigma_small, resolution, relief, vmin, vmax):
    h, w = elev.shape
    dev = elev.device
    s = L.current_stream_ptr()
    stats = torch.empty(3, dtype=torch.int32, device=dev)
    L.check(L.lib().tdx_relief_stats(_p(elev), h * w, _p(stats), s))
    has_nan = int(stats[0]) > 0
    fill = nanmedian_fill(elev) if has_nan else 0.0
    blurred = gaussian_filter(elev, (sigma_large, sigma_small), nan_fill=fill if has_nan else None)
    # Python-float scalars exactly as the reference forms them (relief_map.py:102-103,113,116-117,142-143,168)
    az_deg = float(azimuths[0]) if isinstance(azimuths, (tuple, list)) and len(azimuths) > 0 else 315.0
    alt = np.deg2rad(ALTITUDE_DEG)
    user_range = vmin is not None and vmax is not None
    lo, hi = (max(0.0, float(vmin)), float(vmax)) if user_range else (0.0, 1.0)
    out = torch.empty((h, w, 3), dtype=torch.float32, device=dev)
    L.check(L.lib().tdx_relief_shade(_p(elev), _p(blurred), _p(stats), _p(_lut_on(dev)), h, w, int(has_nan), fill,
                                     15 * resolution / 90, float(np.deg2rad(az_deg)), float(np.sin(alt)),
                                     float(np.cos(alt)), float(relief), 1 - relief, int(user_range), lo,
                                     hi - lo + 1e-8, int(lo == 0.0), _p(out), s))
    return out
