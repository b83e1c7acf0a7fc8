"""The batch-invariant latent stage without a GPU: `WorldPipeline(latents_batch_invariant=)` / `TerrainPipeline`
validation, the option's absence from config.json, `latent_stage_tiles(batch_invariant=True)` argument errors (raised
before any device work), the anchored launch plans of the base model (recorded on the host, tests/_capture.py), the
program cache keys and the ctypes declaration of tdx_latent_embed."""
import json

import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import TerrainPipeline, WorldPipeline, samplers, stages
from terrain_diffusion_b200.inference.solve import DiffusionSolve
from terrain_diffusion_b200.inference.stages import LATENT_BATCH_SIZES, latent_stage_tiles
from terrain_diffusion_b200.inference.tiling import padded_batch_size
from terrain_diffusion_b200.models.plan import UNetEmitter
from tests import test_abi_decl_cpu as ABI
from tests._capture import BASE_CFG, COARSE_CFG, RecordingEmitter, RecordingProgram, folded

BAD = [0, 1, "True", "false", None, 1.0, [True]]


# ------------------------------------------------------------------------------------------------ the option
@pytest.mark.parametrize("bad", BAD)
def test_non_bool_raises_in_the_world_constructor(bad):
    with pytest.raises(ValueError, match="latents_batch_invariant"):
        WorldPipeline(seed=1, latents_batch_invariant=bad)


def _terrain(**kw):
    return TerrainPipeline(None, None, None, 1, coarse_means=[0.0] * 6, coarse_stds=[1.0] * 6, cond_snr=[1.0] * 5,
                           histogram_raw=[0.0] * 5, latents_means=[0.0] * 7, latents_stds=[1.0] * 7, **kw)


@pytest.mark.parametrize("bad", BAD)
def test_non_bool_raises_in_the_terrain_constructor(bad):
    with pytest.raises(ValueError, match="latents_batch_invariant"):
        _terrain(latents_batch_invariant=bad)


@pytest.mark.parametrize("value", [False, True])
def test_bool_values_are_kept(value):
    assert WorldPipeline(seed=1, latents_batch_invariant=value).latents_batch_invariant is value


def test_default_is_off():
    assert WorldPipeline(seed=1).latents_batch_invariant is False


def test_the_option_is_keyword_only():
    import inspect
    for cls in (WorldPipeline, TerrainPipeline):
        p = inspect.signature(cls.__init__).parameters["latents_batch_invariant"]
        assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False


def test_latents_batch_invariant_is_kept_out_of_the_config(tmp_path):
    assert "latents_batch_invariant" in WorldPipeline.ignore_for_config
    WorldPipeline(seed=1, latents_batch_invariant=True).save_pretrained(tmp_path)
    cfg = json.loads((tmp_path / "config.json").read_text())
    assert "latents_batch_invariant" not in cfg
    assert WorldPipeline(**cfg, seed=1).latents_batch_invariant is False


# ------------------------------------------------------------------------------------------------ latent_stage_tiles
class _Recorder:
    """Stands in for the base model and records every step towards device work: reading the model's device, a library
    launch, a program, a noise draw or an embedding launch."""

    def __init__(self, monkeypatch, config=BASE_CFG):
        self.calls = []
        self.config = dict(config)
        monkeypatch.setattr(stages.L, "call", lambda *a, **k: self.calls.append("launch"))
        monkeypatch.setattr(stages, "get_consistency_solve", lambda *a, **k: self.calls.append("program"))
        monkeypatch.setattr(stages, "gaussian_noise_patches", lambda *a, **k: self.calls.append("noise"))
        monkeypatch.setattr(stages, "latent_embedding", lambda *a, **k: self.calls.append("embed"))

    @property
    def device(self):
        self.calls.append("device")
        return torch.device("cpu")


def _args(model, n_ctx, n_cond, n_samples=None, cond_shape=(7, 4, 4), sample_shape=(6, 64, 64), hist=None, **kw):
    samples = None if n_samples is None else [torch.zeros(sample_shape) for _ in range(n_samples)]
    return dict(model=model, seed=0, ctxs=[(0, i, -i) for i in range(n_ctx)], samples=samples,
                cond_imgs=[torch.ones(cond_shape) for _ in range(n_cond)], t=1.0, weight_window=torch.ones(64, 64),
                histogram_raw=torch.zeros(1, 5) if hist is None else hist, cond_means=torch.zeros(7),
                cond_stds=torch.ones(7), batch_invariant=True, **kw)


def _raises(rec, match, **kw):
    with pytest.raises(ValueError, match=match):
        latent_stage_tiles(**kw)
    assert rec.calls == []


@pytest.mark.parametrize("n_ctx,n_cond", [(2, 1), (1, 2), (0, 1), (16, 15)])
def test_mismatched_tiles_and_coarse_windows_raise_before_device_work(monkeypatch, n_ctx, n_cond):
    rec = _Recorder(monkeypatch)
    _raises(rec, "coarse windows", **_args(rec, n_ctx, n_cond))


@pytest.mark.parametrize("n_samples", [1, 3])
def test_mismatched_tiles_and_samples_raise_before_device_work(monkeypatch, n_samples):
    rec = _Recorder(monkeypatch)
    _raises(rec, "samples", **_args(rec, 2, 2, n_samples))


def test_partly_missing_samples_raise_before_device_work(monkeypatch):
    rec = _Recorder(monkeypatch)
    kw = _args(rec, 2, 2, 2)
    kw["samples"][1] = None
    _raises(rec, "all None", **kw)


@pytest.mark.parametrize("top", [None, 16, 4, 1])
def test_more_tiles_than_the_anchor_raise_before_device_work(monkeypatch, top):
    rec = _Recorder(monkeypatch)
    limit = top or LATENT_BATCH_SIZES[-1]
    _raises(rec, f"at most {limit}", **_args(rec, limit + 1, limit + 1, pad_batch_to=top))


@pytest.mark.parametrize("shape", [(6, 4, 4), (7, 4, 5), (7, 16), (1, 7, 4, 4)])
def test_wrong_coarse_window_shape_raises_before_device_work(monkeypatch, shape):
    rec = _Recorder(monkeypatch)
    _raises(rec, r"coarse windows must be \[7, 4, 4\]", **_args(rec, 2, 2, cond_shape=shape))


@pytest.mark.parametrize("shape", [(5, 64, 64), (6, 64, 32), (7, 64, 64)])
def test_wrong_sample_shape_raises_before_device_work(monkeypatch, shape):
    rec = _Recorder(monkeypatch)
    _raises(rec, r"samples must be \[6, 64, 64\]", **_args(rec, 2, 2, 2, sample_shape=shape))


def test_per_tile_histograms_raise_before_device_work(monkeypatch):
    rec = _Recorder(monkeypatch)
    _raises(rec, "one shared histogram", **_args(rec, 2, 2, hist=torch.zeros(2, 5)))


@pytest.mark.parametrize("change", [dict(fourier_scale=1), dict(conditional_inputs=[["float", 58, 1.0]]),
                                    dict(conditional_inputs=[["tensor", 58, 1.0]] * 2), dict(conditional_inputs=[]),
                                    dict(emb_channels=2048), dict(noise_emb_dims=0)])
def test_other_embedding_configurations_raise_before_device_work(monkeypatch, change):
    rec = _Recorder(monkeypatch, dict(BASE_CFG, **change))
    _raises(rec, "batch-invariant latent stage", **_args(rec, 2, 2))


def test_the_coarse_model_is_not_a_latent_model(monkeypatch):
    rec = _Recorder(monkeypatch, COARSE_CFG)
    _raises(rec, "batch-invariant latent stage", **_args(rec, 1, 1))


def test_no_tiles_no_work(monkeypatch):
    rec = _Recorder(monkeypatch)
    assert latent_stage_tiles(**_args(rec, 0, 0)) == []
    assert rec.calls == []


def test_the_shipped_base_model_is_supported():
    spec = stages.latent_embed_spec(type("M", (), {"config": BASE_CFG})())
    assert spec == dict(noise_dims=192, emb_channels=768, cond_dims=58, w_noise=1.0, w_cond=1.0,
                        w_norm=float(torch.linalg.vector_norm(torch.ones(2))))


# ------------------------------------------------------------------------------------------------ launch plans
def recorded(n, batch_invariant, plan_images=1):
    """The igemm descriptors of one base-model forward on n 64^2 tiles, recorded on the host."""
    fw = folded("base")
    prog = RecordingProgram()
    em = RecordingEmitter(fw, n, 64, 64, prog)
    em.batch_invariant, em.plan_images = batch_invariant, plan_images
    meta = torch.device("meta")
    em.emit_embed(prog, emb_in=torch.empty((n, fw.emb_channels), device=meta))
    x = torch.empty((n, fw.in_channels, 64, 64), device=meta)
    em.emit(prog, [(x, fw.in_channels, None)], model_out=torch.empty((n, fw.out_channels, 64, 64), device=meta))
    return prog.igemm()


PADDED = sorted({padded_batch_size(k, LATENT_BATCH_SIZES[-1]) for k in range(1, LATENT_BATCH_SIZES[-1] + 1)})


@pytest.mark.parametrize("anchor", [1, LATENT_BATCH_SIZES[-1]])
def test_anchored_base_plans_force_the_anchor_shape(anchor):
    """Every launch of an anchored batch-invariant forward carries the (N, ksplit) of the free plan at the anchor, at
    every padded batch size, and the library reports exactly that shape (this host's fallback occupancy: the GPU tests
    repeat it with the H100's)."""
    assert PADDED == list(LATENT_BATCH_SIZES)
    plain = [L.igemm_launch_shape(d) for d in recorded(anchor, False)]
    assert len(plain) == 80
    for n in PADDED:
        descs = recorded(n, True, anchor)
        assert [(int(d.n_per_item), int(d.ksplit)) for d in descs] == plain, n
        assert [L.igemm_launch_shape(d) for d in descs] == plain, n


def test_plan_images_must_be_positive():
    with pytest.raises(ValueError, match="plan_images"):
        UNetEmitter(folded("base"), 1, 64, 64, batch_invariant=True, plan_images=0)


def test_plan_images_needs_a_batch_invariant_solve():
    with pytest.raises(ValueError, match="plan_images"):
        DiffusionSolve(object(), None, 2, 64, 64, 1, coef_rows=[{}], plan_images=16)


# ------------------------------------------------------------------------------------------------ program cache keys
class _KeyModel:
    def folded(self):
        return self


@pytest.mark.parametrize("kw,suffix", [({}, ()), (dict(batch_invariant=True), ("batch_invariant",)),
                                       (dict(batch_invariant=True, plan_images=16),
                                        ("plan_images", 16, "batch_invariant"))])
def test_the_program_key_grows_only_with_the_new_options(monkeypatch, kw, suffix):
    built = []
    monkeypatch.setattr(samplers, "DiffusionSolve", lambda *a, **k: built.append(k) or object())
    model = _KeyModel()
    samplers.get_consistency_solve(model, 4, 64, 64, 1.25, 0.5, from_unit_noise=True, out_scale=2.0, **kw)
    (key,) = list(samplers._solve_cache(model))
    assert key == ("cm", 4, 64, 64, 1.25, 0.5, True, 2.0, id(model)) + suffix
    assert built[0]["plan_images"] == kw.get("plan_images", 1)


# ------------------------------------------------------------------------------------------------ the C entry point
def test_ctypes_declaration_matches_the_header():
    assert "tdx_latent_embed" in ABI.PROTOTYPES
    ABI.test_declaration_matches_header("tdx_latent_embed")
