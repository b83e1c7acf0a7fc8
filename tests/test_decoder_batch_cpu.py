"""The batched decoder stage without a GPU: `WorldPipeline(decoder_batch_size=)` / `TerrainPipeline` validation, the
option's absence from config.json, `decoder_stage_tiles` argument errors (raised before any device work) and the
batch-invariant launch plans of the decoder (recorded on the host, tests/_capture.py)."""
import json

import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import TerrainPipeline, WorldPipeline, stages
from terrain_diffusion_b200.inference.stages import DECODER_BATCH_SIZES, decoder_stage_tiles
from tests._capture import RecordingEmitter, RecordingProgram, folded

BAD = [0, 3, 5, 8, 16, -1, 2.0, 4.0, "4", None]


# ------------------------------------------------------------------------------------------------ the option
@pytest.mark.parametrize("bad", BAD)
def test_illegal_decoder_batch_size_raises_in_the_world_constructor(bad):
    with pytest.raises(ValueError, match="decoder_batch_size"):
        WorldPipeline(seed=1, decoder_batch_size=bad)


def _terrain(**kw):
    return TerrainPipeline(None, None, None, 1, coarse_means=[0.0] * 6, coarse_stds=[1.0] * 6, cond_snr=[1.0] * 5,
                           histogram_raw=[0.0] * 5, latents_means=[0.0] * 7, latents_stds=[1.0] * 7, **kw)


@pytest.mark.parametrize("bad", BAD)
def test_illegal_decoder_batch_size_raises_in_the_terrain_constructor(bad):
    with pytest.raises(ValueError, match="decoder_batch_size"):
        _terrain(decoder_batch_size=bad)


@pytest.mark.parametrize("size", DECODER_BATCH_SIZES)
def test_legal_decoder_batch_sizes(size):
    assert DECODER_BATCH_SIZES == (1, 2, 4)
    assert WorldPipeline(seed=1, decoder_batch_size=size).decoder_batch_size == size


def test_default_is_one_window_at_a_time():
    assert WorldPipeline(seed=1).decoder_batch_size == 1


def test_decoder_batch_size_is_kept_out_of_the_config(tmp_path):
    assert "decoder_batch_size" in WorldPipeline.ignore_for_config
    WorldPipeline(seed=1, decoder_batch_size=4).save_pretrained(tmp_path)
    cfg = json.loads((tmp_path / "config.json").read_text())
    assert "decoder_batch_size" not in cfg
    assert WorldPipeline(**cfg, seed=1).decoder_batch_size == 1


# ------------------------------------------------------------------------------------------------ decoder_stage_tiles
class _Recorder:
    """Stands in for the model and records every step towards device work: reading the model's device, a library
    launch, a program or a noise draw."""

    def __init__(self, monkeypatch):
        self.calls = []
        monkeypatch.setattr(stages.L, "call", lambda *a, **k: self.calls.append("launch"))
        monkeypatch.setattr(stages, "get_consistency_solve", lambda *a, **k: self.calls.append("program"))
        monkeypatch.setattr(stages, "gaussian_noise_patches", lambda *a, **k: self.calls.append("noise"))

    @property
    def device(self):
        self.calls.append("device")
        return torch.device("cpu")


def _args(model, n_ctx, n_lat, tile=128, shape=None):
    shape = shape or (6, tile // 8, tile // 8)
    return dict(model=model, seed=0, ctxs=[(0, i, -i) for i in range(n_ctx)],
                latents_windows=[torch.zeros(shape) for _ in range(n_lat)], weight_window=torch.ones(tile, tile),
                t_list=[1.0], tile_size=tile, tile_stride=tile * 3 // 4)


@pytest.mark.parametrize("n_ctx,n_lat", [(2, 1), (1, 2), (0, 1), (4, 3)])
def test_mismatched_windows_and_latents_raise_before_device_work(monkeypatch, n_ctx, n_lat):
    rec = _Recorder(monkeypatch)
    with pytest.raises(ValueError, match="latent windows"):
        decoder_stage_tiles(**_args(rec, n_ctx, n_lat))
    assert rec.calls == []


def test_more_windows_than_the_largest_batch_raise_before_device_work(monkeypatch):
    rec = _Recorder(monkeypatch)
    top = DECODER_BATCH_SIZES[-1]
    with pytest.raises(ValueError, match=f"at most {top}"):
        decoder_stage_tiles(**_args(rec, top + 1, top + 1))
    assert rec.calls == []


@pytest.mark.parametrize("shape", [(5, 16, 16), (6, 16, 15), (6, 64, 64), (6, 16), (1, 6, 16, 16)])
def test_wrong_latent_window_shape_raises_before_device_work(monkeypatch, shape):
    rec = _Recorder(monkeypatch)
    with pytest.raises(ValueError, match=r"latent windows must be \[6, 16, 16\]"):
        decoder_stage_tiles(**_args(rec, 2, 2, shape=shape))
    assert rec.calls == []


def test_wrong_stacked_latent_shape_raises_before_device_work(monkeypatch):
    rec = _Recorder(monkeypatch)
    kw = _args(rec, 3, 3, tile=512)
    kw["latents_windows"] = torch.zeros(3, 6, 32, 32)
    with pytest.raises(ValueError, match=r"latent windows must be \[6, 64, 64\]"):
        decoder_stage_tiles(**kw)
    assert rec.calls == []


def test_no_windows_no_work(monkeypatch):
    rec = _Recorder(monkeypatch)
    assert decoder_stage_tiles(**_args(rec, 0, 0)) == []
    assert rec.calls == []


# ------------------------------------------------------------------------------------------------ launch plans
def recorded(n, hw, batch_invariant):
    """The igemm descriptors of one decoder forward on n hw^2 windows, recorded on the host."""
    fw = folded("decoder")
    prog = RecordingProgram()
    em = RecordingEmitter(fw, n, hw, hw, prog)
    em.batch_invariant = batch_invariant
    meta = torch.device("meta")
    em.emit_embed(prog, labels=torch.empty((n,), device=meta))
    x = torch.empty((n, fw.in_channels, hw, hw), device=meta)
    em.emit(prog, [(x, fw.in_channels, None)], model_out=torch.empty((n, fw.out_channels, hw, hw), device=meta))
    return prog.igemm()


@pytest.mark.parametrize("hw", [128, 512])
def test_batch_invariant_decoder_plans_force_the_one_window_shape(hw):
    """Every launch of a batch-invariant decoder forward carries the (N, ksplit) of its one-window launch at every
    padded batch size, and the library reports exactly that shape (this host's fallback occupancy: the GPU tests
    repeat it with the H100's)."""
    plain = [L.igemm_launch_shape(d) for d in recorded(1, hw, False)]
    for n in DECODER_BATCH_SIZES:
        descs = recorded(n, hw, True)
        assert [(int(d.n_per_item), int(d.ksplit)) for d in descs] == plain, n
        assert [L.igemm_launch_shape(d) for d in descs] == plain, n
