"""The consistency-base and coarse evaluation samplers without a GPU: the fp32 oracle (oracle/eval_samplers.py)
against the reference's own samplers (tests/golden/eval_golden.npz, written by tests/golden/make_golden_eval.py), and
the argument errors of sample_base_consistency / sample_coarse_tiled, which are raised before any device work (the
models here live on the CPU, where any device work would fail with TdxError instead)."""
from __future__ import annotations

import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import eval_samplers as oeval  # noqa: E402
from oracle import scheduler as osched  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from terrain_diffusion_b200.inference import sample_base_consistency, sample_coarse_tiled  # noqa: E402
from terrain_diffusion_b200.models import EDMUnet2D  # noqa: E402
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler  # noqa: E402
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG  # noqa: E402

G = np.load(ROOT / "tests" / "golden" / "eval_golden.npz")


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def _fn(cfg, seed=0):
    sd = ounet.procedural_state_dict(cfg, seed=seed)
    return lambda x, t, c=(): ounet.unet_forward(sd, cfg, x, t, list(c))


def base_case(case):
    """(shape, cond_img, kwargs, unit noise per phase) of a golden base-consistency case."""
    cond = torch.from_numpy(G[f"{case}.cond_img"])
    kw = dict(cond_means=G["bc.means"], cond_stds=G["bc.stds"], noise_level=torch.from_numpy(G[f"{case}.noise_level"]),
              histogram_raw=torch.from_numpy(G[f"{case}.hist"]), intermediate_t=float(G["bc.intermediate_t"]))
    if case == "bc1":
        shape = (2, 5, 64, 64)
        g = torch.Generator().manual_seed(int(G["bc1.noise_seed"]))
        noise = [torch.randn(shape, generator=g) for _ in range(2)]
    else:
        shape = (1, 5, 96, 96)
        noise = list(torch.from_numpy(G["bc96.noise"]))
    return shape, cond, kw, noise


def coarse_draws(cond_img, cond_seed, tile_seed, n_tiles, out_channels, tile):
    """The coarse sampler's draws in the reference's order: randn_like(cond_img) from the global generator, then one
    randn per tile from the generator."""
    torch.manual_seed(cond_seed)
    cond_noise = torch.randn_like(cond_img)
    g = torch.Generator().manual_seed(tile_seed)
    b = cond_img.shape[0]
    return cond_noise, [torch.randn((b, out_channels, tile, tile), generator=g) for _ in range(n_tiles)]


# ------------------------------------------------------------------------------------------------ oracle vs golden
@pytest.mark.slow
@pytest.mark.parametrize("case", ["bc1", "bc96"])
def test_base_consistency_oracle_matches_reference(case):
    shape, cond, kw, noise = base_case(case)
    sch = osched.OracleScheduler()
    sch.set_timesteps(1)
    y = oeval.sample_base_consistency(_fn(BASE_CFG), sch.sigmas[0], 0.5, shape, cond, tile_size=64, noise=noise, **kw)
    assert rel_rms(y, torch.from_numpy(G[f"{case}.y"])) < 1e-5


def test_coarse_oracle_matches_reference():
    cond_img, cond_snr = torch.from_numpy(G["coarse1.cond_img"]), torch.from_numpy(G["coarse1.cond_snr"])
    cond_noise, tile_noise = coarse_draws(cond_img, int(G["coarse1.cond_seed"]), int(G["coarse1.tile_seed"]), 1, 6, 64)
    y = oeval.sample_coarse_tiled(_fn(COARSE_CFG), osched.OracleScheduler, cond_img, cond_snr,
                                  steps=int(G["coarse1.steps"]), tile_size=64, tile_stride=64, out_channels=6,
                                  cond_noise=cond_noise, tile_noise=tile_noise)
    assert rel_rms(y, torch.from_numpy(G["coarse1.y"])) < 1e-5


def test_goldens_are_not_vacuous():
    for case in ("bc1", "bc96", "coarse1"):
        assert float(np.std(G[f"{case}.y"])) > 0.05
        assert 0 < float(G[f"{case}.ref_bf16_err"]) < 0.1
    assert np.isnan(G["bc1.cond_img"][0, 0]).any()


# ------------------------------------------------------------------------------------------------ argument errors
TINY_BASE = dict(image_size=16, in_channels=5, out_channels=5, model_channels=16, model_channel_mults=[1],
                 layers_per_block=1, attn_resolutions=[], midblock_attention=False, concat_balance=0.5,
                 conditional_inputs=[["tensor", 58, 1.0]], fourier_scale="pos")
TINY_COARSE = dict(TINY_BASE, in_channels=11, out_channels=6, conditional_inputs=[["float", 16, 0.2]] * 5)


def _base_call(shape, cond, **kw):
    m = EDMUnet2D(**TINY_BASE).eval()
    args = dict(cond_means=np.zeros(7, np.float32), cond_stds=np.ones(7, np.float32), histogram_raw=torch.zeros(1, 5),
                intermediate_t=0.61, tile_size=64)
    args.update(kw)
    return sample_base_consistency(m, EDMDPMSolverMultistepScheduler(), shape, cond, **args)


def test_base_consistency_needs_a_tile_size():
    with pytest.raises(ValueError, match="tile_size"):
        _base_call((1, 5, 64, 64), torch.zeros(1, 7, 4, 4), tile_size=None)


def test_base_consistency_rejects_a_vector_for_several_tiles():
    with pytest.raises(ValueError, match="must be a tensor image for tiled sampling.*width 5 and height 5"):
        _base_call((1, 5, 96, 96), torch.zeros(58))


@pytest.mark.parametrize("hw", [(4, 4), (5, 4), (6, 6)])
def test_base_consistency_rejects_a_wrongly_sized_cond_image(hw):
    with pytest.raises(ValueError, match="needs 5x5"):
        _base_call((1, 5, 96, 96), torch.zeros(1, 7, *hw))


def test_base_consistency_rejects_too_few_noise_phases():
    with pytest.raises(ValueError, match="noise has 1 phases"):
        _base_call((1, 5, 64, 64), torch.zeros(1, 7, 4, 4), noise=[torch.zeros(1, 5, 64, 64)])


@pytest.mark.parametrize("snr_shape,batch", [((5,), 1), ((2, 5), 2), ((1, 4), 1), ((1, 1, 5), 1)])
def test_coarse_rejects_cond_snr_shapes_the_reference_cannot_run(snr_shape, batch):
    m = EDMUnet2D(**TINY_COARSE).eval()
    with pytest.raises(ValueError, match="cond_snr must be"):
        sample_coarse_tiled(m, EDMDPMSolverMultistepScheduler(), torch.zeros(batch, 5, 64, 64),
                            torch.full(snr_shape, 0.5), steps=2)


def test_coarse_rejects_a_bad_image_or_tile():
    m = EDMUnet2D(**TINY_COARSE).eval()
    with pytest.raises(ValueError, match="cond_img must be"):
        sample_coarse_tiled(m, EDMDPMSolverMultistepScheduler(), torch.zeros(5, 64, 64), torch.full((1, 5), 0.5))
    with pytest.raises(ValueError, match="larger than"):
        sample_coarse_tiled(m, EDMDPMSolverMultistepScheduler(), torch.zeros(1, 5, 48, 64), torch.full((1, 5), 0.5))


def test_cond_inputs_from_snr_matches_the_oracle():
    from terrain_diffusion_b200.inference.samplers import cond_inputs_from_snr
    snr = torch.tensor([[0.1, 0.5, 0.7, 1.5, 3.0]])
    got = cond_inputs_from_snr(snr, "cpu", torch.float32)
    want = oeval.cond_inputs_from_snr(snr)
    assert len(got) == 5 and all(g.shape == (1,) and torch.equal(g, w) for g, w in zip(got, want))


# ------------------------------------------------------------------------------------------------ bench tool
def test_eval_bench_tool_declares_the_evaluation_workload():
    sys.path.insert(0, str(ROOT / "tools"))
    import bench
    import bench_eval_samplers as be
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_eval_samplers.py"), "--help"],
                         capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--images" in out.stdout
    assert (be.EVAL_IMAGES, be.EVAL_TILE, be.EVAL_INTERMEDIATE_T) == (40, 64, 0.61)
    assert be.GFLOP_PER_STEP == bench.GFLOP_PER_LATENT_PHASE == 193.65
