"""The evaluation drivers' terrain decode without a GPU: the fp32 oracle (oracle/eval_terrain.py) against the reference's
own `_decode_latents_to_terrain` (tests/golden/eval_terrain_golden.npz, written by
tests/golden/make_golden_eval_terrain.py), `normalize_uint8_three_channel` against the reference's, and the argument
errors of decode_latents_to_terrain, which are raised before any device work."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import eval_terrain as oterrain  # noqa: E402
from oracle import scheduler as osched  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from terrain_diffusion_b200 import _lib as L  # noqa: E402
from terrain_diffusion_b200.inference import decode_latents_to_terrain, normalize_uint8_three_channel  # noqa: E402
from terrain_diffusion_b200.models import EDMUnet2D  # noqa: E402
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler  # noqa: E402

G = np.load(ROOT / "tests" / "golden" / "eval_terrain_golden.npz")
CASES = ("a", "b", "c", "d")


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def case_inputs(case):
    """(samples, unit noise, inter_t, denoise) of a golden case; the noise is the reference's own CPU draw."""
    samples = torch.from_numpy(G[f"{case}.samples"])
    B, _, h, w = samples.shape
    noise = torch.randn((B, 1, 8 * h, 8 * w), generator=torch.Generator().manual_seed(int(G[f"{case}.noise_seed"])))
    return samples, noise, [float(t) for t in G[f"{case}.inter_t"]], bool(G[f"{case}.denoise"])


class Stats:
    """The dataset attributes decode_latents_to_terrain reads."""

    def __init__(self, **drop):
        self.latents_mean = torch.from_numpy(G["latents_mean"]).view(1, 4, 1, 1)
        self.latents_std = torch.from_numpy(G["latents_std"]).view(1, 4, 1, 1)
        self.residual_mean, self.residual_std = float(G["residual_mean"]), float(G["residual_std"])
        for k in drop:
            delattr(self, k)


class Wrapped:
    def __init__(self, base):
        self.base_dataset = base


# ------------------------------------------------------------------------------------------------ oracle vs golden
@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference(case):
    samples, noise, inter_t, denoise = case_inputs(case)
    sd = ounet.procedural_state_dict(ounet.DECODER_CFG, seed=0)
    sch = osched.OracleScheduler()
    sch.set_timesteps(1)
    y = oterrain.decode_latents_to_terrain(lambda x, t: ounet.unet_forward(sd, ounet.DECODER_CFG, x, t, []),
                                           float(sch.sigmas[0]), 0.5, samples, torch.from_numpy(G["latents_mean"]).view(
                                               1, 4, 1, 1), torch.from_numpy(G["latents_std"]).view(1, 4, 1, 1),
                                           float(G["residual_mean"]), float(G["residual_std"]), noise, inter_t, denoise)
    want = torch.from_numpy(G[f"{case}.y"])
    assert y.shape == want.shape
    assert rel_rms(y, want) < 1e-5


def test_goldens_are_not_vacuous():
    for case in CASES:
        y = G[f"{case}.y"]
        assert float(np.std(y)) > 1.0 and np.isfinite(y).all()
        assert 0 < float(G[f"{case}.ref_bf16_err"]) < 0.05
    assert {G[f"{c}.samples"].shape[-1] for c in CASES} == {8, 16}
    assert {len(G[f"{c}.inter_t"]) for c in CASES} == {0, 1}
    assert {bool(G[f"{c}.denoise"]) for c in CASES} == {False, True}


def test_normalize_uint8_three_channel_matches_reference():
    images = torch.from_numpy(G["uint8.images"])
    want = torch.from_numpy(G["uint8.y"])
    assert torch.equal(normalize_uint8_three_channel(images), want)
    assert torch.equal(oterrain.normalize_uint8_three_channel(images), want)


# ------------------------------------------------------------------------------------------------ argument errors
TINY_DEC = dict(image_size=16, in_channels=5, out_channels=1, model_channels=16, model_channel_mults=[1],
                layers_per_block=1, attn_resolutions=[], midblock_attention=False, concat_balance=0.5,
                conditional_inputs=[], fourier_scale="pos")


def _call(samples, ds=None, **kw):
    return decode_latents_to_terrain(samples, ds if ds is not None else Stats(), EDMUnet2D(**TINY_DEC).eval(),
                                     EDMDPMSolverMultistepScheduler(), torch.Generator(), [0.13], **kw)


@pytest.mark.parametrize("shape", [(2, 4, 8, 8), (5, 8, 8), (2, 6, 8, 8), (0, 5, 8, 8)])
def test_rejects_bad_shapes(shape):
    with pytest.raises(ValueError, match="samples must be|latents"):
        _call(torch.zeros(shape))


@pytest.mark.parametrize("hw", [(8, 12), (12, 16), (4, 8), (9, 9)])
def test_rejects_sizes_that_are_not_multiples_of_8(hw):
    with pytest.raises(ValueError, match="multiples of 8"):
        _call(torch.zeros(1, 5, *hw))


def test_rejects_images_higher_than_wide():
    with pytest.raises(ValueError, match="must fit the width"):
        _call(torch.zeros(1, 5, 16, 8))


def test_rejects_cpu_samples():
    with pytest.raises(L.TdxError, match="CUDA"):
        _call(torch.zeros(1, 5, 8, 8))


@pytest.mark.parametrize("drop", ["latents_mean", "latents_std", "residual_mean", "residual_std"])
def test_rejects_a_dataset_without_its_statistics(drop):
    with pytest.raises(AttributeError, match=drop):
        _call(torch.zeros(1, 5, 8, 8), Stats(**{drop: True}))
    with pytest.raises(AttributeError, match=drop):
        _call(torch.zeros(1, 5, 8, 8), Wrapped(Stats(**{drop: True})))


def test_the_generator_is_untouched_by_a_rejected_call():
    g = torch.Generator().manual_seed(3)
    before = g.get_state()
    with pytest.raises(L.TdxError):
        decode_latents_to_terrain(torch.zeros(1, 5, 8, 8), Stats(), EDMUnet2D(**TINY_DEC).eval(),
                                  EDMDPMSolverMultistepScheduler(), g, [0.13])
    assert torch.equal(g.get_state(), before)
