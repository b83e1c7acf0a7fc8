"""Mirror of the sampling part of terrain_diffusion.inference / terrain_diffusion.training.evaluation."""
from .canvas import BlendCanvas  # noqa: F401
from .samplers import (decode_autoencoder_latents_tiled, sample_autoencoder_tiled,  # noqa: F401
                       sample_base_consistency, sample_base_diffusion, sample_coarse_tiled,
                       sample_decoder_consistency_tiled, sample_decoder_diffusion_sharded,
                       sample_decoder_diffusion_tiled)
from .sharded import ShardedCanvas  # noqa: F401
from .solve import DiffusionSolve, fold_score_scaling  # noqa: F401
from .tiling import linear_weight_window, padded_batch_size, shard_rows, tile_starts, window_range  # noqa: F401
from .stages import (coarse_epilogue, coarse_geometry, coarse_stage_tile, decoder_stage_tile,  # noqa: F401
                     latent_stage_tiles, process_latent_conditioning)
from .lazy_canvas import LazyCanvas, TensorWindow  # noqa: F401
from .pipeline import TerrainPipeline, WorldPipeline  # noqa: F401
from .relief import get_relief_map  # noqa: F401
from .hydrology import d8_flow, flow_accumulation, plot_flow_indicator  # noqa: F401
from .multiphase import (build_timestep_ranges, infinite_diffusion_canvases, phase_step_ranges,  # noqa: F401
                         sample_infinite_diffusion)
