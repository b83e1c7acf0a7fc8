"""The implicit-GEMM shape surface: every forward (model, batch, tile size) the package launches, the places that launch
it, and its igemm launches grouped by (plan class, epilogue signature).

The launch plan (work-item width, split-K, ring depth, cluster, rounds per CTA, partial last round, overlapped or serial
epilogue) depends on the batch as much as on the layer, so the surface follows the batch sizes the code runs:

  * WorldPipeline with its default configuration: the latent stage at every padded batch of `latents_batch_size`, the
    decoder stage on one `decoder_tile_size` tile, the coarse stage on one tile;
  * bench.py: 1 and 16 decoder tiles of 256^2;
  * the evaluation scripts: 40 tiles of the guided base diffusion and of the base consistency sampler, main model and
    guide (tools/bench_guided.py, tools/bench_eval_samplers.py);
  * the tiled samplers' `tile_batch`: the decoder on 256^2 and 512^2 tiles, base, guide, coarse, and the autoencoder's
    encoder on 512^2 tiles and decoder on 64^2 latents, each at every batch up to TILE_BATCH_MAX;
  * PRODUCT, the hand-picked forwards earlier versions of the fp64 replay covered (kept: the surface is a superset).

Recording needs no GPU (tests/_capture.py); planning a launch (`plan_of`) asks the device for its SM count and cluster
occupancy, so `launches()` runs on the GPU.
"""
from __future__ import annotations

import dataclasses
import functools
import inspect
from typing import NamedTuple

import torch

from oracle import autoencoder as oae
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference.pipeline import WorldPipeline
from terrain_diffusion_b200.inference.stages import COARSE_TILE, LATENT_TILE
from terrain_diffusion_b200.inference.tiling import padded_batch_size
from terrain_diffusion_b200.models import EDMAutoencoder
from terrain_diffusion_b200.models.plan import FoldedWeights, autoencoder_decoder_plan
from tests._capture import CONFIGS, capture_forward, layer_of
from tests._igemm_ref import Case, case_from_desc, plan_class, plan_label, plan_of, plan_variant, variant_label
from tests.test_autoencoder_cpu import _record

PRODUCT = [
    # (source, model, batch, tile size)
    ("bench_tiles1", "decoder", 1, 256),           # bench.py (decoder solve, 256^2 tiles)
    ("bench_tiles16", "decoder", 16, 256),
    ("world_decoder_b1", "decoder", 1, 512),       # decoder windows of 512 (WorldPipeline: 1, tiled samplers: 8, 16)
    ("world_decoder_b8", "decoder", 8, 512),
    ("world_decoder_b16", "decoder", 16, 512),
    ("decoder_64", "decoder", 1, 64),
    ("decoder_128_b2", "decoder", 2, 128),
    ("latent_b1", "base", 1, 64),                  # latent stage, batches 1-16 of 64^2 tiles
    ("latent_b2", "base", 2, 64),
    ("latent_b16", "base", 16, 64),
    ("guided_main_b40", "base", 40, 64),           # guided base diffusion: 40 tiles, main model and guide
    ("guide_b16", "guide", 16, 64),
    ("guided_guide_b40", "guide", 40, 64),
    ("coarse_b1", "coarse", 1, 64),
    ("coarse_b16", "coarse", 16, 64),
]

BENCH_TILE, BENCH_TILES = 256, (1, 16)        # bench.py: --size 256, --tiles 1 (default) and 16
EVAL_TILES = 40                               # guided base diffusion and base consistency evaluation batches
DECODER_TILES = (256, 512)                    # the decoder samplers' tile sizes: bench.py and WorldPipeline
AE_TILE = 512                                 # the autoencoder's evaluation tiles (8 x 8 latents per 64 pixels)
TILE_BATCH_MAX = {"decoder": 16, "base": 40, "guide": 40, "coarse": 16, "ae_encoder": 8, "ae_decoder": 8}


class Forward(NamedTuple):
    model: str      # a tests/_capture.py model, or "ae_encoder" / "ae_decoder" (EDMAutoencoder, oracle X8_CFG)
    n: int          # images per launch
    hw: int         # input side: pixels, latents for ae_decoder


def world_pipeline_forwards() -> list:
    """[(source, Forward)] of a WorldPipeline built with its default arguments: the latent stage pads every batch of n
    windows to padded_batch_size(n, max(latents_batch_size)) and prebuilds every listed size; the decoder and coarse
    stages solve one tile at a time."""
    params = inspect.signature(WorldPipeline.__init__).parameters
    sizes = params["latents_batch_size"].default
    sizes = [sizes] if isinstance(sizes, int) else sorted(sizes)
    batches = sorted(set(sizes) | {padded_batch_size(n, sizes[-1]) for n in range(1, sizes[-1] + 1)})
    out = [(f"world_latent_b{m}", Forward("base", m, LATENT_TILE)) for m in batches]
    out.append(("world_decoder_b1", Forward("decoder", 1, params["decoder_tile_size"].default)))
    out.append(("world_coarse_b1", Forward("coarse", 1, COARSE_TILE)))
    return out


def tiled_sampler_forwards() -> list:
    """[(source, Forward)] of the tiled samplers at every `tile_batch` up to TILE_BATCH_MAX."""
    shapes = [("decoder", hw) for hw in DECODER_TILES] + [("base", LATENT_TILE), ("guide", LATENT_TILE),
                                                           ("coarse", COARSE_TILE), ("ae_encoder", AE_TILE),
                                                           ("ae_decoder", AE_TILE // 8)]
    return [(f"tiled_{model}{hw}_b{n}", Forward(model, n, hw))
            for model, hw in shapes for n in range(1, TILE_BATCH_MAX[model] + 1)]


@functools.lru_cache(maxsize=None)
def surface() -> dict:
    """{Forward: [source, ...]} in a fixed order: every forward the package launches and where it comes from."""
    entries = world_pipeline_forwards()
    entries += [(f"bench_tiles{n}", Forward("decoder", n, BENCH_TILE)) for n in BENCH_TILES]
    entries += [(f"eval_{m}_b{EVAL_TILES}", Forward(m, EVAL_TILES, LATENT_TILE)) for m in ("base", "guide")]
    entries += tiled_sampler_forwards()
    entries += [(source, Forward(m, n, hw)) for source, m, n, hw in PRODUCT]
    out: dict = {}
    for source, f in entries:
        if source not in out.setdefault(f, []):
            out[f].append(source)
    return out


@functools.lru_cache(maxsize=None)
def _autoencoder_folded(part: str) -> FoldedWeights:
    torch.manual_seed(0)
    m = EDMAutoencoder(**oae.X8_CFG).eval()
    meta = torch.device("meta")
    if part == "ae_encoder":
        return FoldedWeights(m.encoder, meta)
    return FoldedWeights(m.decoder_view(), meta, plan=autoencoder_decoder_plan(m._decoder_config()))


def record(f: Forward):
    """The RecordingProgram of one forward (no GPU needed)."""
    if f.model in CONFIGS:
        return capture_forward(f.model, f.n, f.hw)
    if f.model == "ae_encoder":
        return _record(_autoencoder_folded(f.model), f.n, f.hw, f.hw, 1, with_embed=True)[0]
    return _record(_autoencoder_folded(f.model), f.n, f.hw, f.hw, 4, with_embed=False)[0]


class Launch(NamedTuple):
    forward: Forward
    sources: tuple      # every source that runs this forward
    layer: str
    case: Case          # named "<first source>:<layer>"
    plan: dict


@functools.lru_cache(maxsize=None)
def launches() -> tuple:
    """Every igemm launch of the surface, planned on this device (recorded once per session)."""
    out = []
    for f, sources in surface().items():
        prog = record(f)
        for d in prog.igemm():
            layer = layer_of(prog, d)
            c = case_from_desc(d, name=f"{sources[0]}:{layer}")
            out.append(Launch(f, tuple(sources), layer, c, plan_of(c)))
    return tuple(out)


def epilogue_signature(c: Case) -> tuple:
    """Epilogue flags, residual mode, pixel-norm side planes, outputs (kind, spatial), clip on/off, tap pattern."""
    has_resid = bool(c.epi & L.EPI_RESID)
    return (c.epi, c.resid_spatial if has_resid else None, c.resid_pnorm if has_resid else None, c.resid_inv,
            c.rms_out, tuple((k, s) for k, s, _ in c.outs), c.clip > 0, tuple(t for _, t in c.segs))


def signature_label(sig) -> str:
    epi, rsp, rpn, rinv, rms, outs, clip, taps = sig
    parts = ["e" + str(epi)]
    if rsp is not None:
        parts.append(f"r{rsp}{'inv' if rinv else ('pn' if rpn else '')}")
    if rms:
        parts.append("rms")
    parts.append("o" + "".join(f"{k}{s}" for k, s in outs))
    if clip:
        parts.append("clip")
    parts.append("t" + "".join(str(t) for t in taps))
    return ".".join(parts)


def group_key(c: Case, p: dict) -> tuple:
    """The surface's group: (plan variant, epilogue signature).  Overlapped or serial follows from the two."""
    return plan_variant(p), epilogue_signature(c)


def representatives(launches, fine: bool = False) -> list:
    """The smallest launch (fewest MACs) of every (plan class, epilogue signature) group -- with `fine`, of every
    (plan variant, epilogue signature) group -- as a Case named "<class or variant label>-<signature>-<name>".
    `launches`: tuples ending in (case, plan)."""
    groups: dict = {}
    for *_, c, p in launches:
        key = group_key(c, p) if fine else (plan_class(p), epilogue_signature(c))
        if key not in groups or c.macs < groups[key].macs:
            groups[key] = c
    label = variant_label if fine else plan_label
    return [dataclasses.replace(c, name=f"{label(cls)}-{signature_label(sig)}-{c.name}")
            for (cls, sig), c in sorted(groups.items(), key=lambda kv: (kv[0][0], str(kv[0][1])))]


def gpu_tests_selected(config) -> bool:
    """Whether this pytest run executes gpu-marked tests: only then is the surface recorded and planned."""
    if not torch.cuda.is_available():
        return False
    expr = config.getoption("markexpr")
    if not expr:
        return True
    try:
        from _pytest.mark.expression import Expression
        return bool(Expression.compile(expr).evaluate(lambda name, **kw: name == "gpu"))
    except Exception:
        return True


def product_launches() -> list:
    """The launches of the PRODUCT forwards in list order, each case named "<PRODUCT source>:<layer>"."""
    by_forward: dict = {}
    for la in launches():
        by_forward.setdefault(la.forward, []).append(la)
    return [la._replace(case=dataclasses.replace(la.case, name=f"{source}:{la.layer}"))
            for source, m, n, hw in PRODUCT for la in by_forward[Forward(m, n, hw)]]


@functools.lru_cache(maxsize=None)
def product_representatives() -> tuple:
    """representatives(product_launches()): one launch per (plan class, epilogue signature) of the PRODUCT forwards."""
    return tuple(representatives(product_launches()))


@functools.lru_cache(maxsize=None)
def group_representatives() -> tuple:
    """The fewest-MAC launch of every group of the surface (representatives(launches(), fine=True))."""
    return tuple(representatives(launches(), fine=True))


def surface_representatives() -> tuple:
    """The group representatives whose group no PRODUCT representative already replays: with
    product_representatives() they run every group of the surface once (the fp64 replay and the fenced-input test)."""
    done = {group_key(c, plan_of(c)) for c in product_representatives()}
    return tuple(c for c in group_representatives() if group_key(c, plan_of(c)) not in done)


def new_groups() -> dict:
    """{group key: [source, ...] in surface order} for the groups of the surface that no PRODUCT forward reaches on
    this device: what the derived surface adds to the hand-picked list."""
    product = {Forward(m, n, hw) for _, m, n, hw in PRODUCT}
    old = {group_key(la.case, la.plan) for la in launches() if la.forward in product}
    out: dict = {}
    for la in launches():
        key = group_key(la.case, la.plan)
        if key not in old:
            out.setdefault(key, []).extend(s for s in la.sources if s not in out[key])
    return out
