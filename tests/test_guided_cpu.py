"""Two-model guidance without a GPU: the fp32 oracle (oracle/guided.py) against the reference's own guided samplers
(tests/golden/guided_golden.npz), and the host-side score-scaling fold of the fused solve."""
from __future__ import annotations

import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import guided as oguided  # noqa: E402
from oracle import scheduler as osched  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from terrain_diffusion_b200.inference.solve import fold_score_scaling  # noqa: E402
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler  # noqa: E402
from tests.test_oracle_golden import BASE_CFG  # noqa: E402

G = np.load(ROOT / "tests" / "golden" / "guided_golden.npz")
GUIDE_CFG = dict(BASE_CFG, model_channels=128)


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def _fn(cfg, seed):
    sd = ounet.procedural_state_dict(cfg, seed=seed)
    return lambda x, t, c=(): ounet.unet_forward(sd, cfg, x, t, list(c))


def _base_noise(shape):
    sch = osched.OracleScheduler()
    sch.set_timesteps(int(G["base.steps"]))
    return torch.randn(shape, generator=torch.Generator().manual_seed(int(G["base.noise_seed"]))) * sch.sigmas[0]


def _base_kwargs():
    return dict(cond_means=G["base.means"], cond_stds=G["base.stds"], noise_level=torch.from_numpy(G["base.noise_level"]),
                histogram_raw=torch.from_numpy(G["base.hist"]), steps=int(G["base.steps"]),
                guidance_scale=float(G["base.guidance"]))


def test_decoder_guided_score_scaled_oracle_matches_reference():
    y = oguided.sample_decoder_diffusion_tiled(_fn(ounet.DECODER_CFG, 0), osched.OracleScheduler,
                                               torch.from_numpy(G["dec.cond"]), torch.from_numpy(G["dec.noise"]), 64,
                                               64, num_steps=int(G["dec.steps"]), guide_fn=_fn(ounet.DECODER_CFG, 1),
                                               guidance_scale=float(G["dec.guidance"]),
                                               score_scaling=float(G["dec.score_scaling"]))
    assert rel_rms(y, torch.from_numpy(G["dec.y"])) < 1e-5


@pytest.mark.slow
def test_base_untiled_guided_oracle_matches_reference():
    y = oguided.sample_base_diffusion(_fn(BASE_CFG, 0), osched.OracleScheduler, (2, 5, 64, 64),
                                      [torch.from_numpy(G["base.cvec"])], noise=_base_noise((2, 5, 64, 64)),
                                      guide_fn=_fn(GUIDE_CFG, 1), **_base_kwargs())
    assert rel_rms(y, torch.from_numpy(G["base1.y"])) < 1e-5


@pytest.mark.slow
def test_base_tiled_guided_oracle_matches_reference():
    y = oguided.sample_base_diffusion(_fn(BASE_CFG, 0), osched.OracleScheduler, (1, 5, 96, 96),
                                      torch.from_numpy(G["base.cond_img"]), noise=_base_noise((1, 5, 96, 96)),
                                      guide_fn=_fn(GUIDE_CFG, 1), tile_size=64, **_base_kwargs())
    assert rel_rms(y, torch.from_numpy(G["base96.y"])) < 1e-5


def test_goldens_are_not_vacuous():
    for case in ("base1", "base96", "dec"):
        assert float(np.std(G[f"{case}.y"])) > 0.05
        assert 0 < float(G[f"{case}.ref_bf16_err"]) < 0.05


def _step_fp64(row, x, f, x0p):
    x0 = row["c_skip"] * x + row["c_out"] * f
    return row["r"] * x + (1 - row["r"]) * x0 + row["k"] * (x0 - x0p), x0


@pytest.mark.parametrize("alpha", [0.8, 1.2, 2.0])
def test_score_scaling_fold_equals_scale_score_then_step(alpha):
    """fold_score_scaling(row) applied to (x, F) == _scale_score(F, x, sigma) then the unfolded row, in fp64."""
    sch = EDMDPMSolverMultistepScheduler()
    sch.set_timesteps(12)
    order = sch.order_schedule()
    g = torch.Generator().manual_seed(3)
    for i in range(12):
        row = sch.step_coefficients(i, order[i])
        sigma = float(sch.sigmas.double()[i])
        x = torch.randn(4096, generator=g, dtype=torch.float64) * math.sqrt(sigma ** 2 + 0.25)
        f = torch.randn(4096, generator=g, dtype=torch.float64)
        x0p = torch.randn(4096, generator=g, dtype=torch.float64)
        want = _step_fp64(row, x, oguided.scale_score(f, x, torch.tensor(sigma, dtype=torch.float64), 0.5, alpha), x0p)
        got = _step_fp64(fold_score_scaling(row, sigma, 0.5, alpha), x, f, x0p)
        for a, b in zip(got, want):
            assert float((a - b).abs().max()) <= 1e-12 * (1 + float(b.abs().max()))


def test_score_scaling_one_leaves_rows_bitwise_unchanged():
    sch = EDMDPMSolverMultistepScheduler()
    sch.set_timesteps(20)
    order = sch.order_schedule()
    for i in range(20):
        row = sch.step_coefficients(i, order[i])
        assert fold_score_scaling(row, float(sch.sigmas[i]), 0.5, 1.0) == row
