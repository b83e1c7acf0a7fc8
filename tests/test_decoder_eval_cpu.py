"""The decoder evaluations without a GPU: the fp32 oracle (oracle/decoder_eval.py) against the reference's own drivers
(tests/golden/decoder_eval_golden.npz, written by tests/golden/make_golden_decoder_eval.py), the blend window and the
step times against the drivers', and the argument errors of decoder_eval_terrain and padded_terrain, which are raised
before any device work (the generator is not drawn from)."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import decoder_eval as odec  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from terrain_diffusion_b200 import _lib as L  # noqa: E402
from terrain_diffusion_b200.inference import decoder_eval_terrain, linear_weight_window, padded_terrain  # noqa: E402
from terrain_diffusion_b200.inference.evaluation import decoder_eval_times  # noqa: E402
from terrain_diffusion_b200.models import EDMUnet2D  # noqa: E402
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler  # noqa: E402
from tests import _decoder_eval_inputs as I  # noqa: E402

G = np.load(ROOT / "tests" / "golden" / "decoder_eval_golden.npz")
CASES = tuple(I.CASES)


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def sub(x, case):
    k = I.SUBSAMPLE[case]
    return x[:, 0, ::k, ::k]


# ------------------------------------------------------------------------------------------------ oracle vs golden
@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference(case):
    c = I.CASES[case]
    sd = ounet.procedural_state_dict(ounet.DECODER_CFG, seed=0)
    g = torch.Generator().manual_seed(I.GENERATOR_SEED)
    for k, batch in enumerate(I.batches(case)):
        fake, real = odec.decoder_eval_batch(lambda x, t: ounet.unet_forward(sd, ounet.DECODER_CFG, x, t, []),
                                             [float(t) for t in G[f"{case}.t"]], batch["image"],
                                             batch["lowfreq_padded"], batch["cond_img"], g,
                                             residual_mean=I.RESIDUAL_MEAN, residual_std=I.RESIDUAL_STD,
                                             sigma_data=I.SIGMA_DATA, tile_size=c["tile_size"],
                                             tile_stride=c["tile_stride"], crop_size=c["crop"])
        assert rel_rms(sub(fake, case), torch.from_numpy(G[f"{case}.{k}.fake"])) < 1e-5
        assert rel_rms(sub(real, case), torch.from_numpy(G[f"{case}.{k}.real"])) < 1e-6
    assert k + 1 == int(G[f"{case}.batches"])


def test_goldens_are_not_vacuous():
    assert [int(G[f"{c}.batches"]) for c in CASES] == [1, 1, 2, 1]
    assert G["dct.1.fake"].shape[0] == 1 and G["dct.0.fake"].shape[0] == 2      # the last batch is truncated
    assert G["tiled.0.fake"].shape == (1, 512 // 4, 512 // 4)                    # the centre crop
    for c in CASES:
        assert 0 < float(G[f"{c}.ref_bf16_err"]) < 1e-2
        for k in range(int(G[f"{c}.batches"])):
            assert bool(G[f"{c}.{k}.u8_3ch"])
            for part in ("fake", "real"):
                y = G[f"{c}.{k}.{part}"]
                assert np.isfinite(y).all() and float(np.std(y)) > 10.0
                assert len(np.unique(G[f"{c}.{k}.{part}_u8"])) > 50
    assert not np.array_equal(G["dc.0.fake"], G["dc1.0.fake"])


def test_times_are_the_drivers():
    sch = EDMDPMSolverMultistepScheduler()
    for c in CASES:
        want = [float(t) for t in G[f"{c}.t"]]
        assert decoder_eval_times(sch, I.CASES[c]["intermediate_sigma"], I.SIGMA_DATA) == want
    assert len(G["dc1.t"]) == 1 and len(G["dc.t"]) == 2


def test_blend_window_is_the_drivers_get_weights():
    w64 = linear_weight_window(64)
    assert torch.equal(w64.view(torch.int32), torch.from_numpy(G["window64"]).view(torch.int32))
    for T in (64, 128, 512):
        assert I.digest(linear_weight_window(T)) == str(G[f"window_sha.{T}"]), T


# ------------------------------------------------------------------------------------------------ argument errors
TINY_DEC = dict(image_size=16, in_channels=5, out_channels=1, model_channels=16, model_channel_mults=[1],
                layers_per_block=1, attn_resolutions=[], midblock_attention=False, concat_balance=0.5,
                conditional_inputs=[], fourier_scale="pos")


def _inputs(S=128, B=2, C=1, lp=None, cc=4):
    h = S // 8
    return (torch.zeros(B, C, S, S), torch.zeros(B, 1, *(lp or (h + 2, h + 2))), torch.zeros(B, cc, S, S))


def _call(images, lowfreq, cond, g=None, **kw):
    kw = dict(dict(residual_mean=0.0, residual_std=1.1678, tile_size=64, tile_stride=32), **kw)
    return decoder_eval_terrain(EDMUnet2D(**TINY_DEC).eval(), EDMDPMSolverMultistepScheduler(), images, lowfreq, cond,
                                g if g is not None else torch.Generator(), **kw)


@pytest.mark.parametrize("inputs, msg", [
    (_inputs(C=2), "square"), (_inputs(S=124), "square"), ((torch.zeros(2, 1, 128, 64),) + _inputs()[1:], "square"),
    (_inputs(lp=(16, 16)), "lowfreq_padded"), (_inputs()[:2] + (torch.zeros(1, 4, 128, 128),), "cond_img"),
    ((torch.zeros(1, 128, 128),) + _inputs()[1:], "must be"),
], ids=["two-channels", "not-multiple-of-8", "not-square", "lowfreq-unpadded", "cond-batch", "3-d"])
def test_rejects_bad_shapes(inputs, msg):
    with pytest.raises(ValueError, match=msg):
        _call(*inputs)


@pytest.mark.parametrize("geom", [dict(tile_size=256), dict(tile_size=64, tile_stride=96),
                                  dict(tile_size=64, tile_stride=48), dict(tile_size=1, tile_stride=1),
                                  dict(tile_size=64, tile_stride=0)])
def test_rejects_tiles_that_leave_pixels_uncovered(geom):
    with pytest.raises(ValueError, match="uncovered"):
        _call(*_inputs(), **geom)


@pytest.mark.parametrize("kw, msg", [(dict(crop_size=129), "crop_size"), (dict(crop_size=0), "crop_size"),
                                     (dict(tile_batch=0), "tile_batch"), (dict(residual_std=[1.0, 2.0]), "scalar")])
def test_rejects_bad_options(kw, msg):
    with pytest.raises(ValueError, match=msg):
        _call(*_inputs(), **kw)


def test_rejects_cpu_images():
    with pytest.raises(L.TdxError, match="CUDA"):
        _call(*_inputs())


def test_the_generator_is_untouched_by_a_rejected_call():
    g = torch.Generator().manual_seed(3)
    before = g.get_state()
    for bad in (dict(tile_size=256), dict()):          # a ValueError, then the CPU-input TdxError
        with pytest.raises((ValueError, L.TdxError)):
            _call(*_inputs(), g=g, **bad)
    assert torch.equal(g.get_state(), before)


def test_padded_terrain_rejects_cpu_and_bad_shapes():
    with pytest.raises(L.TdxError, match="CPU path"):
        padded_terrain(torch.zeros(2, 128, 128), torch.zeros(2, 18, 18), 0.0, 1.0)
