"""The coarse stage's synthetic conditioning map and FastNoiseLite Perlin noise on the device
(terrain_diffusion/inference/synthetic_map.py:182-271, perlin_transform.py:42-45, world_pipeline.py:821-903).

The reference builds each coarse window's five conditioning channels on the host: five pyfastnoiselite Perlin FBm
fields, each quantile-matched to Earth statistics with `np.interp`, then a climate `finalize` and a signed square root
of the elevation.  Here csrc/tdx_synth.cu does all of it in one launch per window, straight into device memory, and
`fbm_perlin` fills any number of FastNoiseLite planes (the Minecraft read-out's detail and climate noise).

The noise restates FastNoiseLite's published 2-D Perlin + FBm algorithm in fp32 with no fused multiply-adds, on the
assumption that the pyfastnoiselite 0.0.6 wheel was built for baseline x86-64.  It is pinned to the numpy restatement in
oracle/synthetic_map.py, not to pyfastnoiselite output: no such fixture exists here.  Everything after the noise is
pinned to the reference's own code (tests/golden/synthetic_golden.npz).

The statistics (quantile tables, temperature-std fit) are the reference's: pass its JSON cache
(`data/global/synthetic_map_stats.json`) or the mapping it loads.  Computing them from the WorldClim rasters needs
rasterio and data that are not part of this package, so `drop_water_pct`, which only enters that computation, has no
effect here.
"""
from __future__ import annotations

import json
import os
import random
from collections.abc import Mapping

import numpy as np
import torch

from .. import _lib as L

STATS_CACHE_PATH = "data/global/synthetic_map_stats.json"     # synthetic_map.py:17, relative to the working directory
MAX_PLANES = 8                                                 # TDX_FBM_MAX_PLANES
MAX_KNOTS = 512                                                # TDX_SYNTH_MAX_KNOTS
FINALIZE, SQRT0, IMPORT, RAW_INPUT = 1, 2, 4, 8                # TDX_SYNTH_* mode bits
MAX_WINDOWS = 16                                                # TDX_SYNTH_MAX_IMAGES: windows per tdx_synthetic_maps
SCALAR_KEYS = ("a_temp_std", "b_temp_std", "temp_std_p1", "temp_std_p99")


def _int(name, v) -> int:
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
        raise ValueError(f"{name} must be an int, got {v!r}")
    return int(v)


def _device(device) -> torch.device:
    if device is None:
        return torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise L.TdxError(f"the synthetic map runs on a CUDA device, got {device}; there is no CPU path")
    return device if device.index is not None else torch.device("cuda", torch.cuda.current_device())


def _int32(seed: int) -> int:
    """A seed as FastNoiseLite stores it: the low 32 bits as a signed int."""
    seed = int(seed) & 0xFFFFFFFF
    return seed - (1 << 32) if seed >= (1 << 31) else seed


# ------------------------------------------------------------------------------------------------------ statistics
def load_stats(stats=None) -> dict:
    """The reference's in-memory statistics from `stats`: a mapping in that form (`noise_quantiles_k`,
    `base_image_quantiles_k`, `a_temp_std`, `b_temp_std`, `temp_std_p1`, `temp_std_p99`), a path to its JSON cache, or
    None for the cache at STATS_CACHE_PATH as the reference reads it.  Raises FileNotFoundError for a missing cache and
    ValueError for tables the transform cannot use: a noise / data table pair of different lengths (as
    `transform_perlin` does), fewer than 2 or more than 512 knots, a noise table that is not strictly increasing, or a
    value that is not finite."""
    if stats is None or isinstance(stats, (str, os.PathLike)):
        path = STATS_CACHE_PATH if stats is None else os.fspath(stats)
        if not os.path.exists(path):
            raise FileNotFoundError(
                f"synthetic map statistics not found at {path!r}: pass stats= (synthetic_map_stats= for a pipeline) as a "
                "path to the reference's cache or as its mapping; computing them from the WorldClim rasters is not "
                "part of this package")
        with open(path, "r", encoding="utf-8") as f:
            data = json.load(f)
        stats = {k: float(data[k]) for k in SCALAR_KEYS}
        for k, t in enumerate(data["noise_quantile_tables"]):
            stats[f"noise_quantiles_{k}"] = t
        for k, t in enumerate(data["data_quantile_tables"]):
            stats[f"base_image_quantiles_{k}"] = t
    if not isinstance(stats, Mapping):
        raise ValueError(f"stats must be a mapping, a path or None, got {type(stats).__name__}")
    out = {}
    for k in SCALAR_KEYS:
        if k not in stats:
            raise ValueError(f"stats has no {k!r}")
        out[k] = float(stats[k])
        if not np.isfinite(out[k]):
            raise ValueError(f"stats[{k!r}] is not finite")
    for c in range(5):
        nk, dk = f"noise_quantiles_{c}", f"base_image_quantiles_{c}"
        if nk not in stats or dk not in stats:
            raise ValueError(f"stats has no {nk!r} / {dk!r}")
        xp = np.asarray(stats[nk], np.float64).reshape(-1)
        fp = np.asarray(stats[dk], np.float64).reshape(-1)
        if len(xp) != len(fp):
            raise ValueError("Source and target quantiles must have the same length "
                             f"(channel {c}: {len(xp)} and {len(fp)})")
        if not 2 <= len(xp) <= MAX_KNOTS:
            raise ValueError(f"channel {c}: {len(xp)} quantiles, 2..{MAX_KNOTS} supported")
        if not (np.isfinite(xp).all() and np.isfinite(fp).all()):
            raise ValueError(f"channel {c}: quantile tables must be finite")
        if not (np.diff(xp) > 0).all():
            raise ValueError(f"channel {c}: the noise quantiles must be strictly increasing")
        out[nk], out[dk] = xp, fp
    if len({len(out[f"noise_quantiles_{c}"]) for c in range(5)}) != 1:
        raise ValueError("every channel must have the same number of quantiles")
    return out


def noise_seeds(seed=None) -> list:
    """The five generator seeds of make_synthetic_map_factory (synthetic_map.py:183): ((seed or a draw from `random`)
    + k + 1) & 0x7FFFFFFF.  Without a seed (None or 0) each of the five is a separate `random.randint(0, 2**30)` draw,
    as in the reference's list comprehension."""
    return [(int(seed or random.randint(0, 2 ** 30)) + k + 1) & 0x7FFFFFFF for k in range(5)]


# ------------------------------------------------------------------------------------------------------ FBm noise
def fbm_planes(configs, i0: int, j0: int, h: int, w: int, out: torch.Tensor) -> torch.Tensor:
    """One `tdx_fbm_perlin` launch: plane k of out (CUDA fp32 [len(configs), h, w], contiguous) is FastNoiseLite Perlin
    FBm of configs[k] = (seed, frequency, octaves, lacunarity, gain) at x = j0 + c, y = i0 + r."""
    n = len(configs)
    if not 1 <= n <= MAX_PLANES:
        raise ValueError(f"1..{MAX_PLANES} noise planes per launch, got {n}")
    if tuple(out.shape) != (n, h, w) or out.dtype != torch.float32 or not out.is_contiguous() or not out.is_cuda:
        raise ValueError(f"out must be a contiguous CUDA fp32 tensor of shape {(n, h, w)}")
    seeds = np.array([_int32(c[0]) for c in configs], np.int32)
    freq = np.array([c[1] for c in configs], np.float32)
    octaves = np.array([_int("octaves", c[2]) for c in configs], np.int32)
    lac = np.array([c[3] for c in configs], np.float32)
    gain = np.array([c[4] for c in configs], np.float32)
    L.call(L.lib().tdx_fbm_perlin, out.device, n, seeds.ctypes.data, freq.ctypes.data, octaves.ctypes.data,
           lac.ctypes.data, gain.ctypes.data, i0, j0, h, w, out.data_ptr())
    return out


def fbm_perlin(seed: int, frequency: float, octaves: int, lacunarity: float, gain: float, i0: int, j0: int, h: int,
               w: int, device=None) -> torch.Tensor:
    """CUDA fp32 [h, w]: pyfastnoiselite's `FastNoiseLite(seed)` with NoiseType_Perlin, FractalType_FBm and these
    settings, `gen_from_coords` at x = j0 + c, y = i0 + r (the coordinates np.arange(..., dtype=np.float32) forms).
    The seed is taken modulo 2^32 as a C int; the float settings are rounded to fp32 as the library stores them.
    Raises ValueError for a non-integer window, an empty one or octaves outside 1..16."""
    i0, j0, h, w = _int("i0", i0), _int("j0", j0), _int("h", h), _int("w", w)
    if h < 1 or w < 1:
        raise ValueError(f"empty noise window {h} x {w}")
    if not 1 <= _int("octaves", octaves) <= 16:
        raise ValueError(f"octaves must be in 1..16, got {octaves}")
    out = torch.empty((1, h, w), dtype=torch.float32, device=_device(device))
    return fbm_planes([(seed, frequency, octaves, lacunarity, gain)], i0, j0, h, w, out)[0]


# ------------------------------------------------------------------------------------------------------ the map
class SyntheticMap:
    """What make_synthetic_map_factory returns: call it as the reference's `sample_full_synthetic_map(i1, j1, i2, j2)`;
    `.sample_raw` and `.finalize` are its attributes of the same names.  Results are CUDA fp32 tensors on `device`.

    Windows follow the reference exactly, including its reshape: the noise is evaluated at x = i1 + c, y = j1 + r over
    a (j2 - j1, i2 - i1) grid whose row-major values are then read as (i2 - i1, j2 - j1).  For a square window that is
    the transposed grid (out[a, b] at x = i1 + b, y = j1 + a); for a non-square one it is the reference's
    reinterpretation, reproduced as is."""

    def __init__(self, stats, frequency_mult, seed=None, device=None):
        if len(frequency_mult) != 5:
            raise ValueError(f"frequency_mult must have 5 values, got {len(frequency_mult)}")
        self.stats = load_stats(stats)
        self.frequency_mult = [float(v) for v in frequency_mult]
        self.n_knots = len(self.stats["noise_quantiles_0"])
        self._tables_host = np.ascontiguousarray(np.stack(
            [np.stack([self.stats[f"noise_quantiles_{c}"], self.stats[f"base_image_quantiles_{c}"]]) for c in range(5)]))
        st = self.stats
        self._scalars = np.array([st["a_temp_std"], st["b_temp_std"], st["temp_std_p1"], st["temp_std_p99"],
                                  st["temp_std_p99"] - st["temp_std_p1"]], np.float64).astype(np.float32)
        self._freq = np.array([0.05 * m for m in self.frequency_mult], np.float64).astype(np.float32)
        self._tables: dict = {}
        self.device = _device(device) if device is not None else None
        self.reseed(seed)

    def reseed(self, seed=None) -> None:
        """Derive the five generator seeds again, as the reference makes a new factory (`_init_conditioning`)."""
        self.seeds = noise_seeds(seed)
        self._seeds = np.array([_int32(s) for s in self.seeds], np.int32)

    def tables(self, device) -> torch.Tensor:
        """The fp64 [5, 2, n_knots] tables on `device`, uploaded once per device."""
        t = self._tables.get(device)
        if t is None:
            t = self._tables[device] = torch.from_numpy(self._tables_host).to(device)
        return t

    def _launch(self, i0, j0, h, w, mode, device=None, input=None, imports=None) -> torch.Tensor:
        dev = input.device if input is not None else _device(device if device is not None else self.device)
        out = torch.empty((5, h, w), dtype=torch.float32, device=dev)
        raw_input = bool(mode & RAW_INPUT)
        tables = None if raw_input else self.tables(dev)
        ptrs = boxes = defaults = None
        has_default = 0
        if imports is not None:
            ptrs, boxes, defaults, has_default = imports
        L.call(L.lib().tdx_synthetic_map, dev, None if tables is None else tables.data_ptr(), self.n_knots,
               self._seeds.ctypes.data, self._freq.ctypes.data, self._scalars.ctypes.data, i0, j0, h, w,
               None if input is None else input.data_ptr(), mode, ptrs, boxes, defaults, has_default,
               out.data_ptr())
        return out

    def _window(self, i1, j1, i2, j2):
        i1, j1, i2, j2 = _int("i1", i1), _int("j1", j1), _int("i2", i2), _int("j2", j2)
        if i2 <= i1 or j2 <= j1:
            raise ValueError(f"empty window [{i1}, {i2}) x [{j1}, {j2})")
        return i1, j1, i2, j2

    def sample_raw(self, i1, j1, i2, j2, device=None) -> torch.Tensor:
        """fp32 [5, i2 - i1, j2 - j1]: the five quantile-matched noise fields before finalize (the reference returns
        them in fp64; every consumer rounds them to fp32 first, which is what this returns)."""
        i1, j1, i2, j2 = self._window(i1, j1, i2, j2)
        return self._launch(j1, i1, j2 - j1, i2 - i1, 0, device).view(5, i2 - i1, j2 - j1)

    def finalize(self, raw) -> torch.Tensor:
        """synthetic_map.py:232-254 on a [5, ...] raw map (tensor or array, rounded to fp32 first), on its device (CUDA
        tensors) or the default device."""
        t = torch.as_tensor(raw)
        if t.dim() < 1 or t.shape[0] != 5 or t.numel() == 0:
            raise ValueError(f"finalize needs a non-empty [5, ...] map, got shape {tuple(t.shape)}")
        dev = t.device if t.is_cuda else _device(self.device)
        t = t.to(device=dev, dtype=torch.float32).contiguous()
        n = t[0].numel()
        out = self._launch(0, 0, 1, n, RAW_INPUT | FINALIZE, input=t.view(5, 1, n))
        return out.view(t.shape)

    def __call__(self, i1, j1, i2, j2, device=None) -> torch.Tensor:
        """fp32 [5, i2 - i1, j2 - j1]: `sample_full_synthetic_map` -- finalize, then sign(x) sqrt|x| of channel 0."""
        i1, j1, i2, j2 = self._window(i1, j1, i2, j2)
        return self._launch(j1, i1, j2 - j1, i2 - i1, FINALIZE | SQRT0, device).view(5, i2 - i1, j2 - j1)

    def from_noise(self, noise, mode=FINALIZE | SQRT0) -> torch.Tensor:
        """The transform and `mode`'s steps applied to given noise fields (CUDA fp32 [5, h, w]) instead of the
        generators': what a caller with its own noise source (or a test) feeds through the same kernel."""
        noise = noise.to(torch.float32).contiguous()
        if noise.dim() != 3 or noise.shape[0] != 5 or not noise.is_cuda:
            raise ValueError(f"noise must be a CUDA [5, h, w] tensor, got {tuple(noise.shape)}")
        return self._launch(0, 0, noise.shape[1], noise.shape[2], mode & (FINALIZE | SQRT0), input=noise)

    def conditioning(self, ci0: int, ci1: int, cj0: int, cj1: int, imports=None, device=None) -> torch.Tensor:
        """fp32 [5, ci1 - ci0, cj1 - cj0]: the reference WorldPipeline's `_conditioning_model_input` of conditioning
        cells [ci0, ci1) x [cj0, cj1).  Without imports the factory's map at (cj0, ci0, cj1, ci1); with `imports`
        (`device_imports`'s tuple) the raw map with them merged and sign(x) sqrt|x| of channel 0 only.  The import mode
        is defined for square windows (the coarse stage's), as in the reference."""
        if imports is None:
            return self(cj0, ci0, cj1, ci1, device=device)
        return self._launch(ci0, cj0, ci1 - ci0, cj1 - cj0, IMPORT | SQRT0, device, imports=imports[:4])

    def conditioning_windows(self, origins, size: int, imports=None, device=None) -> torch.Tensor:
        """fp32 [n, 5, size, size]: `conditioning(ci0, ci0 + size, cj0, cj0 + size, imports)` for every (ci0, cj0) of
        `origins`, in one launch per 16 windows, each bit-identical to its own call."""
        dev = _device(device if device is not None else self.device)
        size = _int("size", size)
        org = np.array([(_int("ci0", a), _int("cj0", b)) for a, b in origins], np.int64).reshape(-1, 2)
        if size < 1 or len(org) == 0:
            raise ValueError(f"conditioning_windows needs windows and a positive size, got {len(org)} of {size}")
        out = torch.empty((len(org), 5, size, size), dtype=torch.float32, device=dev)
        mode = IMPORT | SQRT0 if imports is not None else FINALIZE | SQRT0
        ptrs, boxes, defaults, has_default = imports[:4] if imports is not None else (None, None, None, 0)
        tables = self.tables(dev)
        for g in range(0, len(org), MAX_WINDOWS):
            chunk = np.ascontiguousarray(org[g:g + MAX_WINDOWS])
            L.call(L.lib().tdx_synthetic_maps, dev, tables.data_ptr(), self.n_knots, self._seeds.ctypes.data,
                   self._freq.ctypes.data, self._scalars.ctypes.data, len(chunk), chunk.ctypes.data, size, size, mode,
                   ptrs, boxes, defaults, has_default, out[g].data_ptr())
        return out


def device_imports(imports: dict, origins: dict, defaults: dict, device) -> tuple:
    """The import tables of tdx_synthetic_map from a pipeline's `custom_conditioning_*` dicts: (pointer array, boxes,
    defaults, default bits, the device rasters that keep the pointers alive)."""
    ptrs = np.zeros(5, np.uint64)
    boxes = np.zeros((5, 4), np.int64)
    dflt = np.zeros(5, np.float32)
    bits, keep = 0, []
    for ch, values in imports.items():
        v = torch.as_tensor(values, dtype=torch.float32).to(device).contiguous()
        keep.append(v)
        ptrs[ch] = v.data_ptr()
        boxes[ch] = (*origins[ch], v.shape[0], v.shape[1])
    for ch, d in defaults.items():
        dflt[ch] = np.float32(d)
        bits |= 1 << ch
    return ptrs.ctypes.data, boxes.ctypes.data, dflt.ctypes.data, bits, (ptrs, boxes, dflt, keep)


def make_synthetic_map_factory(frequency_mult=(1.0, 1.0, 1.0, 1.0, 1.0), seed=None, drop_water_pct=0.0, *, stats=None,
                               device=None) -> SyntheticMap:
    """Drop-in for the reference's make_synthetic_map_factory (synthetic_map.py:182-271) on the device.  `stats` is the
    reference's statistics mapping or a path to its JSON cache; None reads the cache at STATS_CACHE_PATH as the
    reference does (FileNotFoundError when it is missing: the statistics are not computed here).  `drop_water_pct`
    only enters that computation and is accepted for compatibility.  `device` defaults to the current CUDA device."""
    del drop_water_pct
    return SyntheticMap(stats, frequency_mult, seed=seed, device=device)
