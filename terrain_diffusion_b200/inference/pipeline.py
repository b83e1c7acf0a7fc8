"""WorldPipeline -- drop-in for terrain_diffusion.inference.world_pipeline.WorldPipeline (reference
inference/world_pipeline.py:287-372 constructor, :541-565 from_pretrained, :567-623 device / to / bind, :690-712 cache and
context manager, :743-819 seed / SNR / custom conditioning, :961-992 + :1133-1203 + :1244-1270 stage wiring,
:1367-1384 get) whose three stages run on the H100 kernels of this package and whose canvases live in HBM.

Callers (`api.py`, `explorer/server.py`, `tiff_export.py`, `world_generator.py`, `latency.py`) only use
`WorldPipeline.from_pretrained(path, seed=..., latents_batch_size=..., torch_compile=..., dtype=..., caching_strategy=...,
cache_limit=..., **kw)`, `.to(device)`, `.bind(hdf5_file)`, `.get(i1, j1, i2, j2, with_climate)`, the lazy tensors
`.coarse / .latents / .residual` (un-normalised (sum x w, sum w) fp32 CPU tensors, negative indices legal) and the small
state API; all of that is here with the reference's argument names and return conventions.

The synthetic conditioning map of the coarse stage (`synthetic_map.py`: five Perlin FBm fields quantile-matched to
Earth statistics) is built on the device per window when `synthetic_map_stats=` is given: the reference's statistics
cache (`data/global/synthetic_map_stats.json`) or its mapping (see inference/synthetic_map.py; computing the statistics
from the WorldClim rasters is not part of this package).  Imports then follow the reference's semantics (raw units,
merged into the Perlin raw map, no finalize, sign(x) sqrt|x| of channel 0 only).  Alternatively inject
`conditioning_fn(i1, i2, j1, j2) -> [5, i2-i1, j2-j1]` (what `_conditioning_model_input` returns) or provide every
channel through `set_custom_conditioning_import`; with none of them the first coarse tile raises.  Passing both
`conditioning_fn` and `synthetic_map_stats` is a ValueError.  `caching_strategy='indirect'` (HDF5 tile
store) is not implemented -- the window cache is the byte-limited HBM LRU of `LazyCanvas` (`cache_limit`, like the
reference's MemoryTileStore).  `torch_compile` is accepted and ignored: every U-Net evaluation already is one CUDA
graph of hand-written kernels.

`coarse_pooling = p` (1, 2, 4, 8 or 16; world_pipeline.py:909-1016) pools every finished coarse solve by p on the
device, channel 0 by `elev_coarse_pool_mode` and channel 1 by `p5_coarse_pool_mode` ('max', 'min', anything else
averages), channels 2-5 by average, so the coarse canvas has p times fewer cells per axis (windows of (64/p)^2 at a
stride of 48/p) and the latent stage and the climate read-out see coarser terrain.  The windows' conditioning cells and
noise do not change.  Any other value raises ValueError in the constructor (the reference asserts only in `bind()`).

`coarse_batch_size = b` (1, 2, 4, 8 or 16, keyword-only; default 1) solves up to b missing coarse windows per call
(`stages.coarse_stage_tiles`).  Every window is bit-identical to its one-window solve, so the canvas, and everything
read from it, does not depend on b.  It is a serving choice, like `latents_batch_size`, and is not written to
config.json.  Any other value raises ValueError in the constructor.

`decoder_batch_size = b` (one of stages.DECODER_BATCH_SIZES, keyword-only; default 1) does the same for the decoder
stage: up to b missing residual windows per call (`stages.decoder_stage_tiles`), each bit-identical to its one-window
solve.  Its consistency program holds b windows of activations (DESIGN.md section 5 gives the measured memory).

`latents_batch_invariant = True` (keyword-only; default False) solves every latent tile bit-identically to its one-tile
solve (`stages.latent_stage_tiles(batch_invariant=True)`): its embedding row is computed on the device from its own
coarse window and its program is planned at a fixed anchor, the largest `latents_batch_size`.  With it, what a world
reads is a function of seed, configuration and coordinates only, whatever the request order, the cache evictions,
`coarse_batch_size` and `decoder_batch_size`.  The bits depend on the largest `latents_batch_size`, and differ from
those of the default path in the last places.  It is not written to config.json.
"""
from __future__ import annotations

import json
import math
import operator
from pathlib import Path

import numpy as np
import torch

from ..scheduler import EDMDPMSolverMultistepScheduler
from .lazy_canvas import LazyCanvas, TensorWindow
from .stages import (COARSE_BATCH_SIZES, DECODER_BATCH_SIZES, coarse_geometry, coarse_stage_tile, coarse_stage_tiles,
                     decoder_stage_tile, decoder_stage_tiles, latent_embed_spec, latent_plan_images,
                     latent_stage_tiles)
from .tiling import linear_weight_window, padded_batch_size

# seed offsets of the latent stage's noise fields: _build_latent_stage (world_pipeline.py:1133-1203) passes 5819 to the
# init phase and 5820 + i to the i-th T_INTER phase (pinned against the reference source by tests/golden/stages_golden.npz)
LATENT_INIT_SEED_OFFSET = 5819
LATENT_STEP_SEED_OFFSET = 5820
# statistics of the base model's 7 conditioning channels (world_pipeline.py:1137-1138)
COND_INPUT_MEAN = [14.99, 11.65, 15.87, 619.26, 833.12, 69.40, 0.66]
COND_INPUT_STD = [21.72, 21.78, 10.40, 452.29, 738.09, 34.59, 0.47]
DEFAULT_COARSE_MEANS = [-37.67916460232751, 2.22578822145657, 18.030293275011356, 333.8442390481231,
                        1350.1259248456176, 52.444339366764396]
DEFAULT_COARSE_STDS = [39.68515115440358, 3.0981253981231522, 8.940333096712806, 322.25238547630295,
                       856.3430083394657, 30.982620765341043]


def _batch_size(name: str, value, legal: tuple) -> int:
    """`value` as an int if it is one of `legal`, else ValueError (a float or a string is not a batch size)."""
    try:
        size = operator.index(value)
    except TypeError:
        size = None
    if size not in legal:
        raise ValueError(f"{name} must be one of {list(legal)}; got {value!r}")
    return size


class _HostView:
    """What slicing one of the reference's InfiniteTensors returns: the un-normalised window sums as a CPU fp32 tensor
    (`server.py:60`, `world_generator.py:29`, `latency.py:76`).  The canvas itself stays on the GPU."""

    def __init__(self, canvas):
        self.canvas = canvas

    def __getitem__(self, key):
        return self.canvas[key].cpu()


class WorldPipeline:
    COARSE_MODEL_FOLDER = "coarse_model"
    BASE_MODEL_FOLDER = "base_model"
    DECODER_MODEL_FOLDER = "decoder_model"
    config_name = "config.json"
    ignore_for_config = ["seed", "latents_batch_size", "coarse_batch_size", "decoder_batch_size",
                         "latents_batch_invariant", "log_mode", "cache_limit", "caching_strategy", "torch_compile",
                         "dtype"]

    def __init__(self, seed: int | None = None, latents_batch_size=(1, 2, 4, 8, 16), native_resolution: float = 90.0, *,
                 T: int = 2, log_mode: str = "info", torch_compile: bool = False, dtype: str | None = None,
                 latent_compression: int = 8, frequency_mult: list | None = None, drop_water_pct: float = 0.5,
                 cond_snr: list | None = None, coarse_pooling: int = 1, elev_coarse_pool_mode: str = "avg",
                 p5_coarse_pool_mode: str = "avg", residual_mean: float = 0.0, residual_std: float = 1.1678,
                 coarse_means: list | None = None, coarse_stds: list | None = None, caching_strategy: str = "direct",
                 cache_limit: int | None = 100 * 1024 * 1024, onestep_latent: bool = False,
                 decoder_tile_size: int = 512, decoder_tile_stride: int = 384, conditioning_fn=None,
                 synthetic_map_stats=None, coarse_batch_size: int = 1, decoder_batch_size: int = 1,
                 latents_batch_invariant: bool = False, **deprecated_kwargs):
        from .noise import next_seed
        if T not in (1, 2):
            raise ValueError(f"T must be 1 or 2, got {T}")
        if conditioning_fn is not None and synthetic_map_stats is not None:
            raise ValueError("pass either conditioning_fn or synthetic_map_stats, not both")
        coarse_geometry(coarse_pooling)                  # ValueError unless it divides 64 and 48 (world_pipeline.py:969-970)
        coarse_pooling = operator.index(coarse_pooling)
        self.coarse_batch_size = _batch_size("coarse_batch_size", coarse_batch_size, COARSE_BATCH_SIZES)
        self.decoder_batch_size = _batch_size("decoder_batch_size", decoder_batch_size, DECODER_BATCH_SIZES)
        if not isinstance(latents_batch_invariant, bool):
            raise ValueError(f"latents_batch_invariant must be True or False; got {latents_batch_invariant!r}")
        self.latents_batch_invariant = latents_batch_invariant
        self.T = T
        self.seed = (int(seed) & 0xFFFFFFFFFFFFFFFF) if seed is not None else next_seed(None)
        sizes = [latents_batch_size] if isinstance(latents_batch_size, int) else sorted(latents_batch_size)
        self._batch_sizes = sizes
        self.latents_batch_size = sizes[-1]
        self.native_resolution = native_resolution          # metres per pixel (world_pipeline.py:293,331)
        self.latent_compression = self.lc = latent_compression
        self.log_mode, self.torch_compile = log_mode, bool(torch_compile)
        self.caching_strategy, self.cache_limit = caching_strategy, cache_limit
        self.onestep_latent = onestep_latent
        self.decoder_tile_size, self.decoder_tile_stride = decoder_tile_size, decoder_tile_stride
        self.kwargs = {
            "latent_compression": latent_compression, "log_mode": log_mode,
            "frequency_mult": frequency_mult if frequency_mult is not None else [1.5, 3, 3, 3, 3],
            "drop_water_pct": drop_water_pct,
            "cond_snr": cond_snr if cond_snr is not None else [0.3, 0.1, 1.0, 0.1, 1.0],
            "coarse_pooling": coarse_pooling, "elev_coarse_pool_mode": elev_coarse_pool_mode,
            "p5_coarse_pool_mode": p5_coarse_pool_mode,
            "histogram_raw": deprecated_kwargs.get("histogram_raw") or [0.0, 0.0, 0.0, 0.0, 0.0],
            "residual_mean": residual_mean, "residual_std": residual_std,
            "coarse_means": list(coarse_means) if coarse_means is not None else list(DEFAULT_COARSE_MEANS),
            "coarse_stds": list(coarse_stds) if coarse_stds is not None else list(DEFAULT_COARSE_STDS),
        }
        self._dtype = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(dtype)
        self.residual_mean, self.residual_std = residual_mean, residual_std
        self.conditioning_fn = conditioning_fn
        self.cond_input_mean = torch.tensor(deprecated_kwargs.get("cond_input_mean", COND_INPUT_MEAN), dtype=torch.float32)
        self.cond_input_std = torch.tensor(deprecated_kwargs.get("cond_input_std", COND_INPUT_STD), dtype=torch.float32)
        self.t_inter_override = deprecated_kwargs.get("t_inter")
        self.coarse_model = self.base_model = self.decoder_model = None
        self.coarse = self.latents = self.residual = None
        self._canvases: dict = {}
        self.custom_conditioning_imports: dict = {}
        self.custom_conditioning_import_origins: dict = {}
        self.custom_conditioning_default_values: dict = {}
        self._host_views = True
        self._set_cond(self.kwargs["cond_snr"])
        # the device synthesis of the conditioning map (never written to config.json: synthetic_map_stats may be a
        # host path); its five noise seeds derive from the world seed as the reference's `_init_conditioning` does
        self._synthetic = None
        self._synthetic_imports = None
        if synthetic_map_stats is not None:
            from .synthetic_map import SyntheticMap
            self._synthetic = SyntheticMap(synthetic_map_stats, self.kwargs["frequency_mult"], seed=self.seed)

    # ------------------------------------------------------------------ construction (world_pipeline.py:470-565)
    @classmethod
    def from_local_models(cls, coarse_model, base_model, decoder_model, **kwargs) -> "WorldPipeline":
        p = cls(**kwargs)
        p.coarse_model, p.base_model, p.decoder_model = coarse_model, base_model, decoder_model
        p._apply_dtype_and_compile()
        return p

    @classmethod
    def load_config(cls, path, **_unused) -> dict:
        f = Path(path) / cls.config_name
        if not f.exists():
            raise FileNotFoundError(f"{f} not found (offline build: local directories only, no HuggingFace Hub)")
        return {k: v for k, v in json.loads(f.read_text()).items() if not k.startswith("_")}

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, token: str | None = None, **kwargs) -> "WorldPipeline":
        """Pipeline config (config.json) + the three U-Nets from their sub-folders, diffusers layout."""
        from ..models import EDMUnet2D
        config = {**cls.load_config(pretrained_model_name_or_path), **kwargs}
        p = cls(**config)
        p.coarse_model = EDMUnet2D.from_pretrained(pretrained_model_name_or_path, subfolder=cls.COARSE_MODEL_FOLDER)
        p.base_model = EDMUnet2D.from_pretrained(pretrained_model_name_or_path, subfolder=cls.BASE_MODEL_FOLDER)
        p.decoder_model = EDMUnet2D.from_pretrained(pretrained_model_name_or_path, subfolder=cls.DECODER_MODEL_FOLDER)
        p._apply_dtype_and_compile()
        return p

    def save_pretrained(self, save_directory: str) -> None:
        root = Path(save_directory)
        root.mkdir(parents=True, exist_ok=True)
        cfg = {"native_resolution": self.native_resolution, "T": self.T, "onestep_latent": self.onestep_latent,
               "decoder_tile_size": self.decoder_tile_size, "decoder_tile_stride": self.decoder_tile_stride,
               **{k: v for k, v in self.kwargs.items() if k != "log_mode"}}
        (root / self.config_name).write_text(json.dumps(cfg, indent=2))
        for folder, m in ((self.COARSE_MODEL_FOLDER, self.coarse_model), (self.BASE_MODEL_FOLDER, self.base_model),
                          (self.DECODER_MODEL_FOLDER, self.decoder_model)):
            if m is not None:
                m.save_pretrained(root / folder)

    def _apply_dtype_and_compile(self) -> None:
        """eval mode; the GPU path computes in bf16 on the tensor cores with fp32 accumulation whatever `dtype` says,
        so there is nothing to convert or compile (world_pipeline.py:400-430)."""
        for m in (self.coarse_model, self.base_model, self.decoder_model):
            if m is not None:
                m.eval()

    @property
    def device(self):
        for m in (self.coarse_model, self.base_model, self.decoder_model):
            if m is not None:
                return next(m.parameters()).device
        return torch.device("cpu")

    def to(self, device):
        for name in ("coarse_model", "base_model", "decoder_model"):
            m = getattr(self, name)
            if m is not None:
                setattr(self, name, m.to(device))
        return self

    def bind(self, hdf5_file: str | None = None, mode: str = "a", compression: str | None = "gzip",
             compression_opts: int | None = 4):
        """Build the stage hierarchy (world_pipeline.py:587-623, 675-679)."""
        if self.caching_strategy != "direct":
            raise NotImplementedError("caching_strategy='indirect' (HDF5 tile store) is out of the hot-path scope; the "
                                      "window cache is the byte-limited HBM cache (cache_limit)")
        if self.device.type != "cuda":
            from .. import _lib as L
            raise L.TdxError("WorldPipeline (GPU path) needs its models on a CUDA device before bind(); no CPU path")
        self._build_hierarchy()
        if self.torch_compile:
            self._prebuild_programs()
        return self

    def _prebuild_programs(self) -> None:
        """`torch_compile=True` in the reference compiles the models for the configured batch sizes before serving
        (world_pipeline.py:393-398, 421-430).  The equivalent here: build (fold, plan, capture) the consistency
        programs of the latent stage for every padded batch size and both phases, and the decoder / coarse programs, so
        that no `get()` pays a plan build the first time a new batch size turns up (0.3-0.5 s each)."""
        from .samplers import get_consistency_solve, get_diffusion_solve
        sd = 0.5
        if self.base_model is not None:
            phases = [(self.t_init, True)] + ([] if self.onestep_latent else [(self.t_inter, False)])
            if self.latents_batch_invariant:
                # the anchored programs at every size latent_stage_tiles pads a batch to
                top = self.latents_batch_size
                latent_embed_spec(self.base_model)
                for m in sorted({padded_batch_size(k, top) for k in range(1, top + 1)}):
                    for t, first in phases:
                        get_consistency_solve(self.base_model, m, 64, 64, float(t), sd, from_unit_noise=first,
                                              out_scale=1.0 / sd, batch_invariant=True,
                                              plan_images=latent_plan_images(top)).prog.instantiate()
            else:
                for m in self._batch_sizes:
                    for t, first in phases:
                        get_consistency_solve(self.base_model, int(m), 64, 64, float(t), sd, from_unit_noise=first,
                                              out_scale=1.0 / sd).prog.instantiate()
        if self.decoder_model is not None:
            T_ = self.decoder_tile_size
            get_consistency_solve(self.decoder_model, 1, T_, T_, float(self.t_init), sd, from_unit_noise=True,
                                  out_scale=1.0 / sd).prog.instantiate()
            for m in (m for m in DECODER_BATCH_SIZES if 1 < m <= self.decoder_batch_size):
                get_consistency_solve(self.decoder_model, m, T_, T_, float(self.t_init), sd, from_unit_noise=True,
                                      out_scale=1.0 / sd, batch_invariant=True).prog.instantiate()
        if self.coarse_model is not None:
            get_diffusion_solve(self.coarse_model, EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80,
                                                                                   sigma_data=0.5), 1, 64, 64,
                                20).prog.instantiate()
            for m in (m for m in COARSE_BATCH_SIZES if 1 < self.coarse_batch_size and m <= self.coarse_batch_size):
                get_diffusion_solve(self.coarse_model, EDMDPMSolverMultistepScheduler(
                    sigma_min=0.002, sigma_max=80, sigma_data=0.5), m, 64, 64, 20, batch_invariant=True).prog.instantiate()

    # ------------------------------------------------------------------ conditioning (injected; see module docstring)
    def _set_cond(self, cond_snr) -> None:
        self.cond_snr = torch.as_tensor(cond_snr, dtype=torch.float32)
        self._t_cond = torch.atan(self.cond_snr)
        self._cond_inputs = [v.view(-1) for v in torch.log(torch.tan(self._t_cond) / 8.0)]

    def set_custom_conditioning_import(self, channel: int, values, origin_i: int, origin_j: int,
                                       default_value: float | None = None) -> None:
        """Install a 2-D raster for conditioning channel 0..4, `values[0, 0]` anchored at conditioning cell
        (origin_i, origin_j); outside its footprint the channel keeps the synthesised value unless `default_value` is
        given (world_pipeline.py:781-819).  With `synthetic_map_stats` the reference's semantics hold: the raster is in
        raw units, merged into the Perlin raw map, and then only channel 0 goes through sign(x) sqrt|x| (no finalize);
        the raster is copied to the device once.  With `conditioning_fn` it is overlaid on that function's output as
        is, in MODEL-INPUT units.  Calls rebuild()."""
        values = np.asarray(values, dtype=np.float32)
        if values.ndim != 2:
            raise ValueError("Custom conditioning import must be a 2-D array.")
        channel = int(channel)
        if not 0 <= channel < 5:
            raise ValueError("channel must be in 0..4")
        self.custom_conditioning_imports[channel] = torch.from_numpy(values.copy())
        self.custom_conditioning_import_origins[channel] = (int(origin_i), int(origin_j))
        if default_value is None:
            self.custom_conditioning_default_values.pop(channel, None)
        else:
            self.custom_conditioning_default_values[channel] = float(default_value)
        self._synthetic_imports = None
        self.rebuild()

    def rebuild(self) -> None:
        """Drop every cached window (world_pipeline.py:714-741; call after changing seed / kwargs that affect tiles).
        With `synthetic_map_stats`, the five noise seeds are derived again from the world seed (a seed of 0 draws new
        ones from `random`, as the reference's `_init_conditioning` does)."""
        if self._synthetic is not None:
            self._synthetic.reseed(self.seed)
        self.empty_cache()

    def _conditioning_model_input(self, i1: int, i2: int, j1: int, j2: int) -> torch.Tensor:
        """[5, i2-i1, j2-j1] raw conditioning map of coarse cells [i1,i2) x [j1,j2) (what the reference's
        `_conditioning_model_input` returns): the injected function, with imported rasters overlaid."""
        if self._synthetic is not None:
            return self._synthetic.conditioning(i1, i2, j1, j2, self._device_imports(), device=self.device)
        covered = all(ch in self.custom_conditioning_default_values for ch in range(5)) and \
            len(self.custom_conditioning_imports) == 5
        if self.conditioning_fn is not None:
            base = torch.as_tensor(self.conditioning_fn(i1, i2, j1, j2), dtype=torch.float32).clone()
        elif covered:
            base = torch.empty((5, i2 - i1, j2 - j1), dtype=torch.float32)
        else:
            raise RuntimeError("no conditioning source: pass conditioning_fn=... (the synthetic-map synthesis of the "
                               "reference is out of scope) or import all 5 channels with default values "
                               "(set_custom_conditioning_import)")
        for ch, arr in self.custom_conditioning_imports.items():
            oi, oj = self.custom_conditioning_import_origins[ch]
            if ch in self.custom_conditioning_default_values:
                base[ch] = self.custom_conditioning_default_values[ch]
            a, b = max(i1, oi), min(i2, oi + arr.shape[0])
            c, d = max(j1, oj), min(j2, oj + arr.shape[1])
            if a < b and c < d:
                base[ch, a - i1:b - i1, c - j1:d - j1] = arr[a - oi:b - oi, c - oj:d - oj]
        return base

    def _device_imports(self):
        """The imported rasters on the device, in tdx_synthetic_map's form (None without imports); copied once after
        each set_custom_conditioning_import."""
        if not self.custom_conditioning_imports:
            return None
        dev = self.device
        if self._synthetic_imports is None or self._synthetic_imports[0] != dev:
            from .synthetic_map import device_imports
            self._synthetic_imports = (dev, device_imports(self.custom_conditioning_imports,
                                                           self.custom_conditioning_import_origins,
                                                           self.custom_conditioning_default_values, dev))
        return self._synthetic_imports[1]

    # ------------------------------------------------------------------ hierarchy (world_pipeline.py:961-1270)
    def _canvas(self, name, *a, **k):
        cv = LazyCanvas(*a, **k)
        self._canvases[name] = cv
        return cv

    def _build_hierarchy(self) -> None:
        dev = self.device
        lim = self.cache_limit
        sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
        self.t_init = math.atan(float(sched.sigmas[0]) / 0.5)
        self.t_inter = math.atan(0.35 / 0.5) if self.t_inter_override is None else float(self.t_inter_override)
        hist = torch.as_tensor(self.kwargs["histogram_raw"], dtype=torch.float32).view(1, -1)
        ww64 = linear_weight_window(64, dev)

        # ---- coarse: 64^2 solves at stride 48, 20-step DPM-Solver++, each pooled by coarse_pooling = p into a
        # (64/p)^2 window at stride 48/p of the coarse canvas
        coarse_sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
        pool = self.kwargs["coarse_pooling"]
        c_tile, c_stride = coarse_geometry(pool)
        ww_coarse = linear_weight_window(c_tile, dev)

        def f_coarse(ctx):
            _, i, j = ctx
            smap = self._conditioning_model_input(i * 48, i * 48 + 64, j * 48, j * 48 + 64)
            return coarse_stage_tile(self.coarse_model, coarse_sched, self.seed, ctx, smap, self._t_cond,
                                     self._cond_inputs, ww_coarse, self.kwargs["coarse_means"],
                                     self.kwargs["coarse_stds"], 20, pool, self.kwargs["elev_coarse_pool_mode"],
                                     self.kwargs["p5_coarse_pool_mode"])

        def f_coarse_batch(ctxs):
            origins = [(i * 48, j * 48) for _, i, j in ctxs]
            if self._synthetic is not None:
                smaps = self._synthetic.conditioning_windows(origins, 64, self._device_imports(), device=self.device)
            else:
                smaps = [self._conditioning_model_input(a, a + 64, b, b + 64) for a, b in origins]
            return coarse_stage_tiles(self.coarse_model, coarse_sched, self.seed, ctxs, smaps, self._t_cond,
                                      self._cond_inputs, ww_coarse, self.kwargs["coarse_means"],
                                      self.kwargs["coarse_stds"], 20, pool, self.kwargs["elev_coarse_pool_mode"],
                                      self.kwargs["p5_coarse_pool_mode"])

        # coarse_batch_size > 1: missing windows are solved up to that many at a time, each bit-identical to its
        # one-window solve (stages.coarse_stage_tiles), so the canvas does not depend on the batching
        batched = self.coarse_batch_size > 1
        coarse = self._canvas("coarse", 7, f_coarse_batch if batched else f_coarse,
                              TensorWindow((7, c_tile, c_tile), (7, c_stride, c_stride)), dev,
                              batch_size=self.coarse_batch_size if batched else None, cache_limit=lim)

        # ---- latents: 64^2 tiles, stride 32; T=2: two consistency phases with a blend in between, T=1: both phases per
        # tile; batches padded to the legal sizes so that only a handful of plans exist.  latents_batch_invariant: each
        # tile is bit-identical to its one-tile solve (stages.latent_stage_tiles), so the canvas does not depend on
        # which tiles were computed together
        out_w = TensorWindow((6, 64, 64), (6, 32, 32))
        coarse_w = TensorWindow((7, 4, 4), (7, 1, 1), (0, -1, -1))
        pad = self.latents_batch_size

        def phase(ctxs, prev, conds, t, off):
            return latent_stage_tiles(self.base_model, self.seed, ctxs, prev, conds, t, ww64, hist, self.cond_input_mean,
                                      self.cond_input_std, seed_offset=off, pad_batch_to=pad,
                                      batch_invariant=self.latents_batch_invariant)

        if self.T == 1:
            def f_t1(ctxs, conds):
                out = phase(ctxs, None, conds, self.t_init, LATENT_INIT_SEED_OFFSET)
                return out if self.onestep_latent else phase(ctxs, out, conds, self.t_inter, LATENT_STEP_SEED_OFFSET)
            latents = self._canvas("latents", 6, f_t1, out_w, dev, args=(coarse,), args_windows=(coarse_w,),
                                   batch_size=pad, cache_limit=lim)
            self._latents_init = latents
        else:
            self._latents_init = latents = self._canvas(
                "latents_init", 6, lambda ctxs, conds: phase(ctxs, None, conds, self.t_init, LATENT_INIT_SEED_OFFSET),
                out_w, dev, args=(coarse,), args_windows=(coarse_w,), batch_size=pad, cache_limit=lim)
            if not self.onestep_latent:
                latents = self._canvas(
                    "latents", 6, lambda ctxs, prev, conds: phase(ctxs, prev, conds, self.t_inter, LATENT_STEP_SEED_OFFSET),
                    out_w, dev, args=(latents, coarse), args_windows=(out_w, coarse_w), batch_size=pad, cache_limit=lim)

        # ---- decoder: T^2 pixel tiles over (T/lc)^2 latent windows, one consistency step
        T_, S_, lc = self.decoder_tile_size, self.decoder_tile_stride, self.lc
        ww_t = linear_weight_window(T_, dev)

        def f_dec(ctx, latents_window):
            return decoder_stage_tile(self.decoder_model, self.seed, ctx, latents_window, ww_t, [self.t_init], T_, S_,
                                      latent_compression=lc)

        def f_dec_batch(ctxs, latents_windows):
            return decoder_stage_tiles(self.decoder_model, self.seed, ctxs, latents_windows, ww_t, [self.t_init], T_,
                                       S_, latent_compression=lc)

        # decoder_batch_size > 1: missing windows are solved up to that many at a time, each bit-identical to its
        # one-window solve (stages.decoder_stage_tiles)
        batched = self.decoder_batch_size > 1
        residual = self._canvas("residual", 2, f_dec_batch if batched else f_dec,
                                TensorWindow((2, T_, T_), (2, S_, S_)), dev, args=(latents,),
                                args_windows=(TensorWindow((6, T_ // lc, T_ // lc), (6, S_ // lc, S_ // lc)),),
                                batch_size=self.decoder_batch_size if batched else None, cache_limit=lim)
        self._coarse, self._latents, self._residual = coarse, latents, residual
        wrap = _HostView if self._host_views else (lambda c: c)
        self.coarse, self.latents, self.residual = wrap(coarse), wrap(latents), wrap(residual)
        self.latents_init = wrap(self._latents_init)

    # ------------------------------------------------------------------ state API (world_pipeline.py:690-779)
    def empty_cache(self) -> None:
        for cv in self._canvases.values():
            cv.clear_cache()

    def change_seed(self, seed: int | None = None) -> bool:
        """New world seed (masked to 64 bits; None draws one like portable_rng.next_seed(None)) and all cached tiles
        dropped; False (no-op) when the seed is unchanged.  With `synthetic_map_stats` the five noise seeds follow the
        new seed; a seed-dependent `conditioning_fn` must read `pipeline.seed` itself."""
        from .noise import next_seed
        new_seed = (int(seed) & 0xFFFFFFFFFFFFFFFF) if seed is not None else next_seed(None)
        if new_seed == self.seed:
            return False
        self.seed = new_seed
        if self._synthetic is not None:
            self._synthetic.reseed(self.seed)
        self.empty_cache()
        return True

    def set_cond_snr(self, cond_snr) -> None:
        if len(cond_snr) != 5:
            raise ValueError("cond_snr must contain exactly 5 values.")
        self.kwargs["cond_snr"] = [float(x) for x in cond_snr]
        self._set_cond(self.kwargs["cond_snr"])
        self.empty_cache()

    def close(self) -> None:
        self.empty_cache()

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc_val, exc_tb):
        self.close()
        return False

    # ------------------------------------------------------------------ read-out (world_pipeline.py:1277-1384)
    def get_elev(self, i1: int, j1: int, i2: int, j2: int, residual_mean: float | None = None,
                 residual_std: float | None = None, as_int16: bool = False):
        """Elevation in metres over pixel rows [i1,i2) x columns [j1,j2), computed on the device (CUDA tensors); with
        as_int16 also the int16 tensor the HTTP API ships (api.py:73-77)."""
        from . import postproc
        mean = self.residual_mean if residual_mean is None else residual_mean
        std = self.residual_std if residual_std is None else residual_std
        if mean is None or std is None:
            raise ValueError("get_elev needs residual_mean / residual_std (constructor or call arguments)")
        return postproc.compute_elev(self._residual, self._latents, i1, j1, i2, j2, self.lc, mean, std,
                                     as_int16=as_int16)

    def _get_device(self, i1, j1, i2, j2, with_climate=True) -> dict:
        from . import postproc
        elev = self.get_elev(i1, j1, i2, j2)
        climate = postproc.compute_climate(self._coarse, i1, j1, i2, j2, elev, self.lc) if with_climate else None
        return {"elev": elev, "climate": climate}

    def get(self, i1: int, j1: int, i2: int, j2: int, with_climate: bool = True) -> dict:
        """{'elev': fp32 [H, W] metres, 'climate': fp32 [5, H, W] | None}, CPU tensors like the reference's."""
        out = self._get_device(i1, j1, i2, j2, with_climate)
        if not self._host_views:
            return out
        return {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in out.items()}

    def get_terrain(self, i1: int, j1: int, i2: int, j2: int, scale: int = 1, with_climate: bool = True) -> dict:
        """The HTTP API's `_get_terrain` (api.py:103-166): {'elev': fp32 [H, W], 'climate': fp32 [5, H, W] | None} over
        rows [i1, i2) x columns [j1, j2) of the world upsampled `scale` times (H = i2 - i1, W = j2 - j1).  The native
        window padded by one pixel is computed on the device and upsampled there, bit for bit with the reference's
        torch CPU bilinear interpolation, at the kept pixels only.  CPU tensors (one pinned copy) for WorldPipeline,
        CUDA tensors for TerrainPipeline.

        Raises ValueError for a non-integer argument, scale < 1 or an empty window at every scale (the reference
        raises for an empty window only at scale 1 and returns wrongly sliced tensors above it)."""
        from . import postproc
        ni1, nj1, ni2, nj2, oi, oj = postproc.terrain_window(i1, j1, i2, j2, scale)
        native = self._get_device(ni1, nj1, ni2, nj2, with_climate)
        out = postproc.upsample_crop(native["elev"], native["climate"], int(scale), oi, oj, i2 - i1, j2 - j1)
        if self._host_views:
            out = postproc.to_host(out)
        return {"elev": out[0], "climate": out[1:] if with_climate else None}

    def terrain_payload(self, i1: int, j1: int, i2: int, j2: int, scale: int = 1) -> tuple:
        """(body, (H, W)) of `GET /terrain` (api.py:174-201): body is `_binary_response(**_get_terrain(...))`'s, byte for
        byte -- int16-LE elevation (floor, clip; NaN packs as 0) followed by climate channels 0..3 as fp32-LE interleaved
        per pixel.  Packed on the device and copied to the host once.  Argument errors as get_terrain."""
        from . import postproc
        ni1, nj1, ni2, nj2, oi, oj = postproc.terrain_window(i1, j1, i2, j2, scale)
        native = self._get_device(ni1, nj1, ni2, nj2, True)
        H, W = i2 - i1, j2 - j1
        body = postproc.upsample_crop(native["elev"], native["climate"], int(scale), oi, oj, H, W, payload=True)
        return postproc.to_host(body).numpy().tobytes(), (H, W)

    def get_minecraft(self, i1: int, j1: int, i2: int, j2: int, scale: int = 1, noise: float = 1.0,
                      noise_fn=None) -> dict:
        """The Minecraft API's read-out (minecraft_api.py `_handle_1x` / `_handle_upsampled` up to the response):
        {'elev', 'elev_smooth': fp32 [H, W], 'climate': fp32 [5, H, W] | None, 'biome': int16 [H, W]} over rows
        [i1, i2) x columns [j1, j2) of the world upsampled `scale` times.  Scale 1 reads the window and, for the slope,
        the window with a 1-pixel ring; scale >= 2 reads the native window padded by 2 pixels, upsamples it bit for bit
        with the reference's torch CPU bilinear interpolation and, for noise > 0, adds the slope-scaled detail noise
        to 'elev' ('elev_smooth' is without it).  'biome' holds the classifier's Minecraft biome ids; all plains when
        there is no climate.  One launch on the device; CPU tensors (pinned copies) for WorldPipeline, CUDA tensors for
        TerrainPipeline.

        `noise_fn(cfg, i0, j0, h, w) -> fp32 [h, w]` supplies the FastNoiseLite noise planes (see inference/minecraft.py);
        it must be a pure function of its arguments.  The default uses pyfastnoiselite and raises RuntimeError without it.
        Raises ValueError for a non-integer window or scale, scale < 1, an empty window, more than 65535 rows or a
        non-numeric `noise`.  The reference fails on a one-column window taller than one row (its Sobel `.squeeze()`
        drops the column axis); here that window is classified like any other."""
        from . import minecraft, postproc
        (planes, biome), _ = minecraft.request(self._get_device, self.native_resolution, i1, j1, i2, j2, scale, noise,
                                               noise_fn, payload=False)
        if self._host_views:
            planes, biome = postproc.to_host(planes), postproc.to_host(biome)
        return {"elev": planes[0], "elev_smooth": planes[1], "climate": planes[2:] if planes.shape[0] == 7 else None,
                "biome": biome}

    def minecraft_payload(self, i1: int, j1: int, i2: int, j2: int, scale: int = 1, noise: float = 1.0,
                          noise_fn=None) -> tuple:
        """(body, (H, W)) of the Minecraft API's binary `GET /terrain`: body is `_binary_response(elev, biome=biome)`'s,
        byte for byte -- int16-LE elevation (floor, clip; NaN packs as 0), then the int16-LE biome ids.  Packed on the
        device and copied to the host once.  Arguments and errors as get_minecraft."""
        from . import minecraft, postproc
        body, hw = minecraft.request(self._get_device, self.native_resolution, i1, j1, i2, j2, scale, noise, noise_fn,
                                     payload=True)
        return postproc.to_host(body).numpy().tobytes(), hw

    def get_relief(self, i1: int, j1: int, i2: int, j2: int, **kw):
        """Shaded relief RGB [H, W, 3] of the elevation over pixel rows [i1,i2) x columns [j1,j2): `get_elev` and then
        `get_relief_map` on the device, with `resolution` defaulting to `native_resolution` as the explorer passes it
        (server.py:219-226).  numpy for WorldPipeline, a CUDA tensor for TerrainPipeline."""
        rgb = self._relief_on_device(i1, j1, i2, j2, **kw)
        return rgb.cpu().numpy() if self._host_views else rgb

    def _relief_on_device(self, i1: int, j1: int, i2: int, j2: int, **kw) -> torch.Tensor:
        from .relief import get_relief_map
        kw.setdefault("resolution", self.native_resolution)
        return get_relief_map(self.get_elev(i1, j1, i2, j2), None, None, None, **kw)

    def get_detail(self, i1: int, j1: int, i2: int, j2: int, mode: str = "relief"):
        """The explorer's `/api/detail.png` picture of pixel rows [i1, i2) x columns [j1, j2) (server.py:188-231) as the
        uint8 RGBA [H, W, 4] that `plt.imsave` hands to the PNG encoder; the caller encodes the PNG.  mode 'elevation':
        the elevation in the `terrain` colormap, from `get_elev` alone (the reference also computes the climate and
        discards it); 'temperature': climate plane 0 in `RdBu_r`; any other mode: the shaded relief of `get_relief`'s
        device path (resolution = native_resolution), NaN pixels transparent.  numpy (one pinned copy) for
        WorldPipeline, a CUDA tensor for TerrainPipeline.

        Raises ValueError before any device work for a non-integer coordinate, an empty window, more than 65535 rows,
        or a relief window narrower than 2 pixels on either axis."""
        from . import explorer, postproc
        explorer.detail_window(i1, j1, i2, j2, mode)
        if mode == "elevation":
            img = explorer.colour_image(self.get_elev(i1, j1, i2, j2), "terrain")
        elif mode == "temperature":
            img = explorer.colour_image(self._get_device(i1, j1, i2, j2, True)["climate"][0], "RdBu_r")
        else:
            img = explorer.relief_rgba8(self._relief_on_device(i1, j1, i2, j2))
        return postproc.to_host(img).numpy() if self._host_views else img

    def detail_raw_payload(self, i1: int, j1: int, i2: int, j2: int) -> tuple:
        """(body, (H, W), has_temp) of the explorer's `GET /api/detail_raw` (server.py:234-270): body is byte for byte
        the handler's -- H*W int16-LE elevations (floor, clip; NaN packs as 0), then climate plane 0 as H*W fp32-LE --
        and has_temp is its X-Has-Temp.  Packed on the device in one launch and copied to the host once.  Argument errors
        as get_detail."""
        from . import explorer, postproc
        H, W = explorer.detail_window(i1, j1, i2, j2)
        out = self._get_device(i1, j1, i2, j2, True)
        temp = out["climate"][0] if out["climate"] is not None else None
        body = explorer.raw_body(out["elev"], temp)
        return postproc.to_host(body).numpy().tobytes(), (H, W), temp is not None

    # ------------------------------------------------------------------ coarse map (explorer/server.py:58-185)
    def _coarse_sums(self, ci0: int, ci1: int, cj0: int, cj1: int) -> torch.Tensor:
        """The coarse canvas slice [7, h, w] of (sum v*w, sum w), on the device."""
        return self._coarse[:, ci0:ci1, cj0:cj1]

    def get_coarse(self, ci0: int, ci1: int, cj0: int, cj1: int, eps: bool = True):
        """fp32 [6, h, w] real-unit planes of coarse cells [ci0, ci1) x [cj0, cj1): v / (w + 1e-8) as the explorer's
        `_coarse_channel` divides (eps=True) or v / w as `normalize_tensor` does (eps=False), then sign(x) * x^2 for
        channels 0 and 1 (metres).  One launch; a CPU tensor (one pinned copy) for WorldPipeline, a CUDA tensor for
        TerrainPipeline.  Raises ValueError before any device work for a non-integer coordinate, an empty window or
        more than 65535 rows."""
        from . import coarse_view as CV, postproc
        CV.coarse_window(ci0, ci1, cj0, cj1)
        planes, _ = CV.readout(self._coarse_sums(ci0, ci1, cj0, cj1), eps)
        return postproc.to_host(planes[:6]) if self._host_views else planes[:6]

    def coarse_image(self, ci0: int, ci1: int, cj0: int, cj1: int, channel: int = 0, filters: dict | None = None,
                     lut=None) -> tuple:
        """(rgba8, vmin, vmax) of the explorer's `GET /api/coarse.png` (server.py:102-146): the uint8 RGBA [h, w, 4]
        that `plt.imsave` hands to the PNG encoder, and the Python floats the handler rounds into X-Vmin / X-Vmax.
        `channel` is shown in `lut` (default: matplotlib's viridis, read once; RuntimeError without matplotlib),
        channel 4 as log1p(max(x, 0)), over its NaN-ignoring range.  `filters` = {channel: (lo | None, hi | None)}
        dims to 0.3 every cell where a given bound fails (`>= lo`, `<= hi`, as numpy compares fp32 with a Python float;
        NaN fails), as the `ch{c}_min` / `ch{c}_max` arguments do; channel 1 is ignored, as in the handler.  Two
        launches; numpy for WorldPipeline, a CUDA tensor for TerrainPipeline.

        Raises ValueError before any device work for a bad window (as get_coarse), an unknown channel, a malformed
        filter or a lut that is not [256, 3]."""
        from . import coarse_view as CV
        CV.coarse_window(ci0, ci1, cj0, cj1)
        channel = CV.check_channel(channel)
        bounds, active = CV.filter_bounds(filters)
        table = CV.check_lut(lut)
        planes, rng = CV.readout(self._coarse_sums(ci0, ci1, cj0, cj1), True)
        img = CV.image(planes, rng, channel, bounds, active, CV.lut_on(table, planes.device))
        if self._host_views:
            img, rng = CV.to_host_all(img, rng)
            img = img.numpy()
        return (img, *CV.display_range(rng, channel))

    def coarse_data(self, ci0: int, ci1: int, cj0: int, cj1: int) -> dict:
        """The dict the explorer's `GET /api/coarse_data.json` passes to `jsonify` (server.py:149-164): the window and
        every channel's `np.round(_coarse_channel(...), 2).tolist()` by name.  Two launches and one copy.  Argument
        errors as get_coarse."""
        from . import coarse_view as CV, postproc
        CV.coarse_window(ci0, ci1, cj0, cj1)
        planes, _ = CV.readout(self._coarse_sums(ci0, ci1, cj0, cj1), True)
        host = postproc.to_host(CV.rounded(planes)).numpy()
        return {"ci0": ci0, "ci1": ci1, "cj0": cj0, "cj1": cj1,
                "channels": {name: host[i].tolist() for i, name in enumerate(CV.CHANNEL_NAMES)}}

    def coarse_stats(self, ci0: int, ci1: int, cj0: int, cj1: int) -> dict:
        """The dict of the explorer's `GET /api/coarse_stats` (server.py:167-185): {channel: {'name', 'min', 'max'}}
        with the NaN-ignoring min and max of each channel rounded to 3 decimals, from one launch and one 56-byte copy.
        Argument errors as get_coarse."""
        from . import coarse_view as CV, postproc
        CV.coarse_window(ci0, ci1, cj0, cj1)
        _, rng = CV.readout(self._coarse_sums(ci0, ci1, cj0, cj1), True, planes=False)
        ranges = CV.range_values(postproc.to_host(rng))
        return {ch: {"name": name, "min": round(ranges[ch][0], 3), "max": round(ranges[ch][1], 3)}
                for ch, name in enumerate(CV.CHANNEL_NAMES)}

    def land_tiles(self, coarse_window: int, detail_size: int, min_land_frac: float = 0.5) -> list:
        """The `valid_tiles` of random_sampler.sample_land_tiles (random_sampler.py:71-93), in its order: every (ci, cj)
        of the coarse window [-coarse_window, coarse_window)^2 whose (2 half)^2 cells around it, half =
        (detail_size // 256) // 2, are at least `min_land_frac` land (elevation > 0 under v / w).  Four launches and one
        copy of the list.  Raises ValueError before any device work unless coarse_window is a positive int and
        detail_size a non-negative int; half == 0 finds nothing, as the reference's empty mean is NaN."""
        from . import coarse_view as CV
        if isinstance(coarse_window, bool) or not isinstance(coarse_window, (int, np.integer)) or coarse_window < 1:
            raise ValueError(f"coarse_window must be a positive int, got {coarse_window!r}")
        cw = int(coarse_window)
        CV.coarse_window(-cw, cw, -cw, cw)
        half = CV.land_half(detail_size)
        min_land_frac = float(min_land_frac)
        planes, _ = CV.readout(self._coarse_sums(-cw, cw, -cw, cw), False)
        return CV.land_positions(planes[0], half, min_land_frac, -cw, -cw)

    def residual_normalized(self, i1: int, j1: int, i2: int, j2: int) -> torch.Tensor:
        """Blended decoder output over pixel rows [i1,i2) x columns [j1,j2): residual[0] / residual[1] (on the device)."""
        r = self._residual[:, i1:i2, j1:j2]
        return r[0] / r[1]


class TerrainPipeline(WorldPipeline):
    """Device-resident variant for callers that stay on the GPU: live models + a conditioning source (an injected
    `conditioning_fn` or `synthetic_map_stats` for the device synthesis) in the constructor, bound immediately,
    `.coarse / .latents / .residual / .get` return CUDA tensors."""

    def __init__(self, coarse_model, base_model, decoder_model, seed: int, conditioning_fn=None, *, coarse_means,
                 coarse_stds,
                 cond_snr, histogram_raw, latents_means, latents_stds, latents_batch_size: int = 16,
                 decoder_tile_size: int = 512, decoder_tile_stride: int = 384, latent_compression: int = 8,
                 t_inter: float | None = None, residual_mean: float | None = None, residual_std: float | None = None,
                 native_resolution: float = 90.0, cache_limit: int | None = None, coarse_pooling: int = 1,
                 elev_coarse_pool_mode: str = "avg", p5_coarse_pool_mode: str = "avg", synthetic_map_stats=None,
                 frequency_mult: list | None = None, coarse_batch_size: int = 1, decoder_batch_size: int = 1,
                 latents_batch_invariant: bool = False):
        super().__init__(seed=seed, latents_batch_size=latents_batch_size, native_resolution=native_resolution,
                         latent_compression=latent_compression, cond_snr=[float(v) for v in cond_snr],
                         coarse_pooling=coarse_pooling, elev_coarse_pool_mode=elev_coarse_pool_mode,
                         p5_coarse_pool_mode=p5_coarse_pool_mode, residual_mean=residual_mean, residual_std=residual_std,
                         coarse_means=[float(v) for v in coarse_means], coarse_stds=[float(v) for v in coarse_stds],
                         cache_limit=cache_limit, decoder_tile_size=decoder_tile_size,
                         decoder_tile_stride=decoder_tile_stride, conditioning_fn=conditioning_fn,
                         synthetic_map_stats=synthetic_map_stats, frequency_mult=frequency_mult,
                         histogram_raw=[float(v) for v in torch.as_tensor(histogram_raw).flatten()],
                         cond_input_mean=[float(v) for v in torch.as_tensor(latents_means).flatten()],
                         cond_input_std=[float(v) for v in torch.as_tensor(latents_stds).flatten()], t_inter=t_inter,
                         coarse_batch_size=coarse_batch_size, decoder_batch_size=decoder_batch_size,
                         latents_batch_invariant=latents_batch_invariant)
        self.coarse_model, self.base_model, self.decoder_model = coarse_model, base_model, decoder_model
        self._host_views = False
        self._build_hierarchy()

    @property
    def device(self):
        return self.decoder_model.device
