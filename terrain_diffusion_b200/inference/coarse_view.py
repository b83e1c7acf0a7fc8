"""The explorer's coarse map and the random sampler's land search on the device (terrain_diffusion/inference/explorer/
server.py:58-185, inference/random_sampler.py:61-119).

`GET /api/coarse.png` shows one coarse channel in `viridis` (channel 4 as log1p), dims the cells that fail the
`ch{c}_min` / `ch{c}_max` filters and sends the range back as `X-Vmin` / `X-Vmax`; `GET /api/coarse_data.json` sends
all six channels rounded to two decimals; `GET /api/coarse_stats` their min and max.  The reference copies the coarse
canvas to the host once per channel it reads and runs numpy / matplotlib there.  The random sampler looks for coarse
tiles whose (2 half)^2 window is mostly land with a Python double loop over the whole coarse window.  Here
csrc/tdx_coarse_view.cu does all of it on the canvas slice in device memory; the caller copies one image, one array,
14 range keys or one tile list to the host.  PNG / JSON encoding stays on the host.

The `viridis` table is not restated: it is 256 listed colours, read once from matplotlib when it is installed (the
explorer's server imports it anyway).  Without matplotlib, pass the table as `lut=`.
"""
from __future__ import annotations

import random

import numpy as np
import torch

from .. import _lib as L
from . import postproc

CHANNEL_NAMES = ["Elev", "p5", "Temp", "T std", "Precip", "Precip CV"]   # server.py:22
FILTERABLE = (0, 2, 3, 4, 5)                                          # server.py:121: p5 is never a filter
LUT_SIZE = 256
N_PLANES = 7                                                          # the six channels + channel 4's display plane
_viridis: dict = {}


def coarse_window(ci0, ci1, cj0, cj1) -> tuple[int, int]:
    """(h, w) of coarse cells [ci0, ci1) x [cj0, cj1); ValueError for a non-integer coordinate, an empty window or more
    than 65535 rows."""
    for name, v in (("ci0", ci0), ("ci1", ci1), ("cj0", cj0), ("cj1", cj1)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError(f"{name} must be an int, got {v!r}")
    h, w = int(ci1) - int(ci0), int(cj1) - int(cj0)
    if h <= 0 or w <= 0:
        raise ValueError(f"empty coarse window: rows [{ci0}, {ci1}) x columns [{cj0}, {cj1})")
    if h > 65535:
        raise ValueError(f"at most 65535 rows, got {h}")
    return h, w


def check_channel(channel) -> int:
    if isinstance(channel, bool) or not isinstance(channel, (int, np.integer)) or not 0 <= int(channel) < 6:
        raise ValueError(f"channel must be an int in 0..5 ({', '.join(CHANNEL_NAMES)}), got {channel!r}")
    return int(channel)


def filter_bounds(filters) -> tuple[np.ndarray, int]:
    """(fp32 [6, 2] bounds, active bits) of `filters` = {channel: (lo | None, hi | None)}.  Each bound is rounded to
    fp32, as numpy does when it compares an fp32 array with a Python float (overflow to inf).  Channel 1 is accepted and
    ignored, as the handler never reads `ch1_*`."""
    bounds, active = np.zeros((6, 2), np.float32), 0
    for ch, pair in (filters or {}).items():
        ch = check_channel(ch)
        try:
            lo, hi = pair
        except (TypeError, ValueError):
            raise ValueError(f"filters[{ch}] must be a (lo | None, hi | None) pair, got {pair!r}") from None
        for side, v in enumerate((lo, hi)):
            if v is None or ch not in FILTERABLE:
                continue
            if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)):
                raise ValueError(f"filters[{ch}] bounds must be numbers or None, got {v!r}")
            with np.errstate(over="ignore"):
                bounds[ch, side] = np.float32(float(v))
            active |= 1 << (2 * ch + side)
    return bounds, active


def check_lut(lut) -> np.ndarray:
    """fp64 [256, 3] RGB table: `lut` (any real [256, 3] array), or viridis from matplotlib when `lut` is None."""
    if lut is None:
        return viridis_lut()
    arr = np.asarray(lut.detach().cpu() if isinstance(lut, torch.Tensor) else lut)
    if arr.shape != (LUT_SIZE, 3) or arr.dtype.kind not in "fiu":
        raise ValueError(f"lut must be a real [{LUT_SIZE}, 3] RGB table, got {arr.dtype} {arr.shape}")
    return arr.astype(np.float64)


def viridis_lut() -> np.ndarray:
    """`plt.get_cmap('viridis')`'s 256 listed colours as fp64 [256, 3], read from the installed matplotlib."""
    if "table" not in _viridis:
        try:
            import matplotlib
        except ImportError:
            raise RuntimeError("coarse_image: the viridis table is read from matplotlib, which is not installed; pass "
                               "lut= (an fp [256, 3] RGB table, e.g. matplotlib.colormaps['viridis'](np.arange(256))"
                               "[:, :3] saved elsewhere)") from None
        cmap = matplotlib.colormaps["viridis"]
        _viridis["table"] = np.asarray(cmap(np.arange(cmap.N)), dtype=np.float64)[:, :3].copy()
    return _viridis["table"]


def check_sums(sums: torch.Tensor) -> torch.Tensor:
    """A coarse canvas slice: CUDA fp32 [7, h, w] of (sum v*w, sum w), made contiguous."""
    if not (isinstance(sums, torch.Tensor) and sums.is_cuda and sums.dtype == torch.float32 and sums.dim() == 3
            and sums.shape[0] == 7 and sums.numel() > 0):
        raise L.TdxError(f"coarse view: expected a non-empty CUDA float32 [7, h, w] canvas slice (the GPU read-out has "
                         f"no CPU path), got {getattr(sums, 'device', None)} {getattr(sums, 'dtype', None)} "
                         f"{tuple(getattr(sums, 'shape', ()))}")
    return sums.contiguous()


def readout(sums: torch.Tensor, eps: bool = True, planes: bool = True):
    """(planes, range) of a canvas slice in one launch: CUDA fp32 [7, h, w] (channels 0..5 in real units -- x = v /
    (w + 1e-8) with eps as `_coarse_channel` divides, v / w without as `normalize_tensor` does, then sign(x) * x^2 for
    channels 0 and 1 -- and log1p(max(channel 4, 0))), or None without `planes`; and the CUDA int32 [14] range keys of
    the seven planes (`range_values` decodes them)."""
    sums = check_sums(sums)
    dev, (_, h, w) = sums.device, sums.shape
    out = torch.empty((N_PLANES, h, w), dtype=torch.float32, device=dev) if planes else None
    rng = torch.empty(2 * N_PLANES, dtype=torch.int32, device=dev)
    L.call(L.lib().tdx_coarse_readout, dev, sums.data_ptr(), h * w, int(bool(eps)),
           None if out is None else out.data_ptr(), rng.data_ptr())
    return out, rng


def _key_to_float(k: int) -> float:
    b = (k & 0x7FFFFFFF) if k & 0x80000000 else (~k & 0xFFFFFFFF)
    return float(np.array(b, np.uint32).view(np.float32))


def range_values(rng) -> list[tuple[float, float]]:
    """[(nanmin, nanmax)] of the seven planes as Python floats (NaN for an all-NaN plane) from readout's range keys."""
    keys = [int(k) & 0xFFFFFFFF for k in np.asarray(rng.cpu() if isinstance(rng, torch.Tensor) else rng).tolist()]
    out = []
    for p in range(N_PLANES):
        nmn, kmx = keys[2 * p], keys[2 * p + 1]
        out.append((_key_to_float(~nmn & 0xFFFFFFFF), _key_to_float(kmx)) if kmx else (float("nan"), float("nan")))
    return out


def display_range(rng, channel: int) -> tuple[float, float]:
    """server.py:113-116: vmin, vmax of the channel's display plane, vmax = vmin + 1 when equal."""
    vmin, vmax = range_values(rng)[6 if channel == 4 else channel]
    if vmax == vmin:
        vmax = vmin + 1
    return vmin, vmax


def lut_on(table: np.ndarray, device: torch.device) -> torch.Tensor:
    """The table rounded to fp32 (the handler's `.astype(np.float32)` of the RGBA) on `device`; viridis is cached."""
    if table is _viridis.get("table"):
        if device not in _viridis:
            _viridis[device] = torch.from_numpy(table.astype(np.float32)).to(device)
        return _viridis[device]
    return torch.from_numpy(table.astype(np.float32)).to(device)


def image(planes: torch.Tensor, rng: torch.Tensor, channel: int, bounds: np.ndarray, active: int,
          lut: torch.Tensor) -> torch.Tensor:
    """The uint8 RGBA [h, w, 4] of `/api/coarse.png` (server.py:112-139) from readout's planes and range (eps on)."""
    dev, (_, h, w) = planes.device, planes.shape
    out = torch.empty((h, w, 4), dtype=torch.uint8, device=dev)
    b = np.ascontiguousarray(bounds, np.float32)
    L.call(L.lib().tdx_coarse_image, dev, planes.data_ptr(), h * w, int(channel), rng.data_ptr(), lut.data_ptr(),
           b.ctypes.data, int(active), out.data_ptr())
    return out


def rounded(planes: torch.Tensor) -> torch.Tensor:
    """np.round(x, 2) of the six real-unit planes (server.py:159): CUDA fp32 [6, h, w]."""
    six = planes[:6]
    out = torch.empty_like(six)
    L.call(L.lib().tdx_coarse_round, planes.device, six.data_ptr(), six.numel(), out.data_ptr())
    return out


def land_half(detail_size) -> int:
    """random_sampler.py:83-84: half = (detail_size // 256) // 2."""
    if isinstance(detail_size, bool) or not isinstance(detail_size, (int, np.integer)) or detail_size < 0:
        raise ValueError(f"detail_size must be a non-negative int, got {detail_size!r}")
    half = (int(detail_size) // 256) // 2
    if half > 2048:
        raise ValueError(f"detail_size {detail_size} covers more than 4096 coarse cells per side")
    return half


def land_positions(elev_m: torch.Tensor, half: int, min_land_frac: float, ci0: int = 0,
                   cj0: int = 0) -> list[tuple[int, int]]:
    """[(ci0 + i, cj0 + j)] for the window centres (i, j), in row-major order, whose land fraction (elev_m > 0 over rows
    [i - half, i + half) x columns [j - half, j + half)) is >= min_land_frac, i in [half, h - half), j in [half, w -
    half); four launches and one copy of the list."""
    elev_m = postproc.check_plane(elev_m, "land_positions")
    dev, (h, w) = elev_m.device, elev_m.shape
    ho, wo = h - 2 * half, w - 2 * half
    n = max(ho, 0) * max(wo, 0)
    rows = torch.empty((h, wo), dtype=torch.int32, device=dev) if n else None
    mask = torch.empty((ho, wo), dtype=torch.uint8, device=dev) if n else None
    lst = torch.empty(1 + n, dtype=torch.int32, device=dev)
    L.call(L.lib().tdx_coarse_land, dev, elev_m.data_ptr(), h, w, half, float(min_land_frac),
           None if rows is None else rows.data_ptr(), None if mask is None else mask.data_ptr(), lst.data_ptr())
    host = postproc.to_host(lst).numpy()
    idx = host[1:1 + int(host[0])].astype(np.int64)
    wo = max(wo, 1)
    return list(zip((ci0 + half + idx // wo).tolist(), (cj0 + half + idx % wo).tolist()))


def to_host_all(*tensors) -> list[torch.Tensor]:
    """Device -> pinned host copies of all `tensors` (one device), on its current stream, with one wait."""
    out = []
    for t in tensors:
        staging = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        staging.copy_(t, non_blocking=True)
        out.append(staging)
    torch.cuda.current_stream(tensors[0].device).synchronize()
    return out


# ---------------------------------------------------------------------------------------- the random sampler's API
def sample_land_tiles(world, coarse_window: int, detail_size: int, min_land_frac: float = 0.5,
                      n_samples: int = 10) -> list:
    """Drop-in for random_sampler.sample_land_tiles: `world.land_tiles` finds every (ci, cj) of the coarse window
    [-coarse_window, coarse_window)^2 whose detail tile is at least `min_land_frac` land, in the reference's order; the
    draw stays on the host and uses the global `random` state, so a seeded run picks the same tiles."""
    valid_tiles = world.land_tiles(coarse_window, detail_size, min_land_frac)
    if len(valid_tiles) < n_samples:
        print(f"Warning: Only found {len(valid_tiles)} valid land tiles (requested {n_samples})")
        return valid_tiles
    return random.sample(valid_tiles, n_samples)


def get_coarse_climate_info(world, ci: int, cj: int) -> dict:
    """Drop-in for random_sampler.get_coarse_climate_info: channels 2..5 of coarse cell (ci, cj) as `normalize_tensor`
    gives them (v / w), as Python floats."""
    planes = world.get_coarse(ci, ci + 1, cj, cj + 1, eps=False)
    vals = planes[2:6, 0, 0].tolist()
    return {"temp": vals[0], "temp_std": vals[1], "precip": vals[2], "precip_cv": vals[3]}
