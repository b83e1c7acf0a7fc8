"""Two-model guided sampling on the GPU: the guided last convolution inside the fused solve, score scaling, the
decoder sampler with a guide and sample_base_diffusion, against the reference's own guided samplers
(tests/golden/guided_golden.npz, written by tests/golden/make_golden_guided.py) and against the public model +
scheduler called step by step.

Tolerance (DESIGN section 2): rel-RMS <= 1.0e-2 vs the reference's fp32 output AND <= 1.25 x the reference's own
bf16-autocast error on the same inputs; where that error alone exceeds 1.0e-2 (guidance amplifies F_m - F_g), only the
second half applies.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import unet as ounet
from terrain_diffusion_b200.inference import DiffusionSolve, sample_base_diffusion, sample_decoder_diffusion_tiled
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests.test_oracle_golden import BASE_CFG

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "guided_golden.npz")
GUIDE_CFG = dict(BASE_CFG, model_channels=128)


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def check_golden(y, case):
    ref = torch.from_numpy(G[f"{case}.y"])
    ref_err = float(G[f"{case}.ref_bf16_err"])
    err = rel_rms(y.float().cpu(), ref)
    assert float(ref.std()) > 0.05
    assert err <= 1.25 * ref_err, (case, err, ref_err)
    if ref_err <= 1.0e-2:
        assert err <= 1.0e-2, (case, err, ref_err)


def build(cfg, seed):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=seed))
    return m.cuda()


@pytest.fixture(scope="module")
def base_pair():
    return build(BASE_CFG, 0), build(GUIDE_CFG, 1)


@pytest.fixture(scope="module")
def decoder_pair():
    return build(ounet.DECODER_CFG, 0), build(ounet.DECODER_CFG, 1)


def _base_kwargs():
    return dict(cond_means=G["base.means"], cond_stds=G["base.stds"],
                noise_level=torch.from_numpy(G["base.noise_level"]), histogram_raw=torch.from_numpy(G["base.hist"]),
                steps=int(G["base.steps"]), guidance_scale=float(G["base.guidance"]))


# ------------------------------------------------------------------------------------------------ goldens
def test_base_untiled_guided_matches_reference(base_pair):
    m, g = base_pair
    y = sample_base_diffusion(m, EDMDPMSolverMultistepScheduler(), (2, 5, 64, 64),
                              [torch.from_numpy(G["base.cvec"])], guide_model=g,
                              generator=torch.Generator().manual_seed(int(G["base.noise_seed"])), **_base_kwargs())
    check_golden(y, "base1")


def test_base_tiled_guided_matches_reference(base_pair):
    m, g = base_pair
    y = sample_base_diffusion(m, EDMDPMSolverMultistepScheduler(), (1, 5, 96, 96),
                              torch.from_numpy(G["base.cond_img"]), guide_model=g, tile_size=64,
                              generator=torch.Generator().manual_seed(int(G["base.noise_seed"])), **_base_kwargs())
    check_golden(y, "base96")


def test_decoder_guided_score_scaled_matches_reference(decoder_pair):
    m, g = decoder_pair
    y = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), torch.from_numpy(G["dec.cond"]).cuda(),
                                       torch.from_numpy(G["dec.noise"]).cuda(), 64, 64, num_steps=int(G["dec.steps"]),
                                       guidance_model=g, guidance_scale=float(G["dec.guidance"]),
                                       score_scaling=float(G["dec.score_scaling"]))
    check_golden(y, "dec")


# ------------------------------------------------------------------------------------------------ fused == unfused
def _scale_score(f, x, sigma, sd, alpha):
    """sample_diffusion_decoder.py:7-40, restated."""
    if alpha == 1.0:
        return f
    v = -sd * f
    t = torch.atan(torch.as_tensor(sigma, dtype=x.dtype, device=x.device) / sd)
    c, s = torch.cos(t), torch.sin(t)
    x0 = x * c - v * s
    npred = x * s + v * c
    x0a = x + alpha * (x0 - x)
    return (npred * c - x0a * s) / -sd


@pytest.mark.parametrize("which", ["decoder_cout1", "base_cout8"])
def test_fused_guided_solve_equals_model_twice_plus_scheduler(which, decoder_pair, base_pair):
    """The one-graph guided solve == the public model and guide called per step, combined on the host, score-scaled
    and stepped with scheduler.step."""
    gen = torch.Generator().manual_seed(21)
    if which == "decoder_cout1":
        (m, g), n, cs, cc, scale, alpha = decoder_pair, 2, 1, 4, 1.5, 1.2
        cond = torch.randn(n, cc, 64, 64, generator=gen).cuda()
        ci = []
    else:
        (m, g), n, cs, cc, scale, alpha = base_pair, 2, 5, 0, 2.15, 1.0
        cond = None
        ci = [torch.randn(n, 58, generator=gen).cuda()]
    noise = (torch.randn(n, cs, 64, 64, generator=gen) * 80).cuda()
    sch = EDMDPMSolverMultistepScheduler()
    solve = DiffusionSolve(m, sch, n, 64, 64, 5, guide=g, guidance_scale=scale, score_scaling=alpha)
    fused = solve.run(noise, cond, conditional_inputs=ci).clone()
    sch.set_timesteps(5)
    x = noise.clone()
    for t, sigma in zip(sch.timesteps, sch.sigmas):
        xin = sch.precondition_inputs(x, sigma)
        if cond is not None:
            xin = torch.cat([xin, cond], dim=1)
        cn = sch.trigflow_precondition_noise(sigma.view(-1).expand(n)).cuda()
        fm, fg = m(xin, cn, ci), g(xin, cn, ci)
        f = _scale_score(fg + scale * (fm - fg), x, sigma, 0.5, alpha)
        x = sch.step(f, t, x).prev_sample
    assert rel_rms(fused, x) < 2e-3


# ------------------------------------------------------------------------------------------------ invariants
def test_guidance_scale_one_is_the_unguided_program(decoder_pair):
    m, g = decoder_pair
    gen = torch.Generator().manual_seed(5)
    noise = (torch.randn(1, 1, 64, 64, generator=gen) * 80).cuda()
    cond = torch.randn(1, 4, 64, 64, generator=gen).cuda()
    a = DiffusionSolve(m, EDMDPMSolverMultistepScheduler(), 1, 64, 64, 4)
    b = DiffusionSolve(m, EDMDPMSolverMultistepScheduler(), 1, 64, 64, 4, guide=g, guidance_scale=1.0)
    assert a.launches_per_solve == b.launches_per_solve
    assert torch.equal(a.run(noise, cond).clone(), b.run(noise, cond).clone())
    ya = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond, noise, 64, 64, num_steps=4)
    yb = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond, noise, 64, 64, num_steps=4,
                                        guidance_model=g, guidance_scale=1.0)
    assert torch.equal(ya, yb)
    guided = DiffusionSolve(m, EDMDPMSolverMultistepScheduler(), 1, 64, 64, 4, guide=g, guidance_scale=1.5)
    assert guided.launches_per_solve == 2 * a.launches_per_solve        # two embeds + two forwards per step


def test_tiled_base_one_tile_at_a_time_matches_reference_and_replays_bitwise(base_pair):
    """Batch size is a free choice: tiles solved one at a time meet the same golden as the batched run (the
    implicit-GEMM kernel picks its work split per batch size, so the two are not bit-identical -- as for the unguided
    solve), and a repeated call is bit-identical."""
    m, g = base_pair

    def run(tb):
        return sample_base_diffusion(m, EDMDPMSolverMultistepScheduler(), (1, 5, 96, 96),
                                     torch.from_numpy(G["base.cond_img"]), guide_model=g, tile_size=64,
                                     generator=torch.Generator().manual_seed(int(G["base.noise_seed"])), tile_batch=tb,
                                     **_base_kwargs())
    check_golden(run(1), "base96")
    assert torch.equal(run(None), run(None))


def test_decoder_sampler_with_guide_and_tile_batch_matches_oracle(decoder_pair):
    from oracle import guided as oguided
    from oracle import scheduler as osched
    m, g = decoder_pair
    sd0, sd1 = (ounet.procedural_state_dict(ounet.DECODER_CFG, seed=s) for s in (0, 1))
    gen = torch.Generator().manual_seed(4)
    noise = torch.randn(1, 1, 96, 96, generator=gen) * 80
    cond = torch.randn(1, 4, 96, 96, generator=gen)
    ref = oguided.sample_decoder_diffusion_tiled(
        lambda x, t: ounet.unet_forward(sd0, ounet.DECODER_CFG, x, t, []), osched.OracleScheduler, cond, noise, 64,
        32, num_steps=3, guide_fn=lambda x, t: ounet.unet_forward(sd1, ounet.DECODER_CFG, x, t, []),
        guidance_scale=1.5, score_scaling=1.2)
    for tb in (1, 4):
        y = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond.cuda(), noise.cuda(), 64, 32,
                                           num_steps=3, guidance_model=g, guidance_scale=1.5, score_scaling=1.2,
                                           tile_batch=tb)
        assert rel_rms(y.cpu(), ref) < 1.0e-2, tb


def test_unplannable_guide_names_the_channel_count(decoder_pair):
    m, _ = decoder_pair
    small = build(dict(ounet.DECODER_CFG, model_channels=32), 1)
    gen = torch.Generator().manual_seed(6)
    noise = (torch.randn(1, 1, 64, 64, generator=gen) * 80).cuda()
    cond = torch.randn(1, 4, 64, 64, generator=gen).cuda()
    with pytest.raises(NotImplementedError, match="32 channels"):
        sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond, noise, 64, 64, num_steps=2,
                                       guidance_model=small, guidance_scale=1.5)
