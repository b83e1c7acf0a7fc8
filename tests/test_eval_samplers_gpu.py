"""sample_base_consistency and sample_coarse_tiled on the GPU: against the reference's own evaluation samplers
(tests/golden/eval_golden.npz, written by tests/golden/make_golden_eval.py), against the fp32 oracle on multi-tile
canvases, and against the public model called per tile and per phase.

Tolerance (DESIGN section 2): rel-RMS <= 1.0e-2 vs the reference's fp32 output AND <= 1.25 x the reference's own
bf16-autocast error on the same inputs; where that error alone exceeds 1.0e-2, only the second half applies.  Each
check prints its error share of the binding bound.
"""
from __future__ import annotations

import math
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import eval_samplers as oeval
from oracle import scheduler as osched
from oracle import unet as ounet
from terrain_diffusion_b200.inference import (process_latent_conditioning, sample_base_consistency,
                                              sample_coarse_tiled)
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests.test_eval_samplers_cpu import base_case, coarse_draws
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "eval_golden.npz")


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def check(y, ref, ref_err, what):
    err = rel_rms(y.float().cpu(), ref)
    assert float(ref.std()) > 0.05
    bound = 1.25 * ref_err if ref_err > 1.0e-2 else min(1.0e-2, 1.25 * ref_err)
    print(f"\n{what}: rel-RMS {err:.3e}, reference bf16 {ref_err:.3e}, share of bound {err / bound:.3f}")
    assert err <= bound, (what, err, ref_err)


def check_golden(y, case):
    check(y, torch.from_numpy(G[f"{case}.y"]), float(G[f"{case}.ref_bf16_err"]), case)


def build(cfg, seed=0):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=seed))
    return m.cuda()


@pytest.fixture(scope="module")
def base():
    return build(BASE_CFG)


@pytest.fixture(scope="module")
def coarse():
    return build(COARSE_CFG)


def run_case(model, case, **extra):
    shape, cond, kw, noise = base_case(case)
    if case == "bc1":
        extra.setdefault("generator", torch.Generator().manual_seed(int(G["bc1.noise_seed"])))
    else:
        extra.setdefault("noise", noise)
    return sample_base_consistency(model, EDMDPMSolverMultistepScheduler(), shape, cond, tile_size=64, **kw, **extra)


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("case", ["bc1", "bc96"])
def test_base_consistency_matches_reference(base, case):
    y = run_case(base, case)
    assert y.shape == base_case(case)[0] and y.is_cuda and y.dtype == torch.float32
    check_golden(y, case)


def test_coarse_one_tile_matches_reference(coarse):
    torch.manual_seed(int(G["coarse1.cond_seed"]))
    y = sample_coarse_tiled(coarse, EDMDPMSolverMultistepScheduler(), torch.from_numpy(G["coarse1.cond_img"]),
                            torch.from_numpy(G["coarse1.cond_snr"]), steps=int(G["coarse1.steps"]),
                            generator=torch.Generator().manual_seed(int(G["coarse1.tile_seed"])))
    assert y.device.type == "cpu" and y.shape == (1, 6, 64, 64)
    check_golden(y, "coarse1")


# ------------------------------------------------------------------------------------------------ multi-tile coarse
def test_coarse_multi_tile_matches_oracle(coarse):
    """112^2 at tile 64 / stride 48: 2x2 tiles with overlaps, each from a reset solver.  The reference-bf16 half of the
    rule comes from the oracle itself run under CPU bf16 autocast."""
    gen = torch.Generator().manual_seed(31)
    cond_img = torch.randn(1, 5, 112, 112, generator=gen)
    cond_snr = torch.tensor([[0.2, 0.5, 1.0, 0.5, 2.0]])
    steps = 3
    cond_noise, tile_noise = coarse_draws(cond_img, 41, 43, 4, 6, 64)
    sd = ounet.procedural_state_dict(COARSE_CFG, seed=0)

    def oracle():
        return oeval.sample_coarse_tiled(lambda x, t, c: ounet.unet_forward(sd, COARSE_CFG, x, t, c),
                                         osched.OracleScheduler, cond_img, cond_snr, steps=steps, tile_size=64,
                                         tile_stride=48, out_channels=6, cond_noise=cond_noise, tile_noise=tile_noise)
    ref = oracle()
    with torch.autocast("cpu", dtype=torch.bfloat16):
        ref16 = oracle().float()
    torch.manual_seed(41)
    y = sample_coarse_tiled(coarse, EDMDPMSolverMultistepScheduler(), cond_img, cond_snr, steps=steps, tile_size=64,
                            tile_stride=48, generator=torch.Generator().manual_seed(43))
    check(y, ref, rel_rms(ref16, ref), "coarse 112^2")


# ------------------------------------------------------------------------------------------------ fused == unfused
def test_fused_consistency_equals_public_model_per_tile_and_phase(base):
    """bc96 (2x2 tiles, two phases) with the public model(...) called per tile and phase, the TrigFlow mixing and the
    blend done with host torch ops on the device."""
    shape, cond, kw, noise = base_case("bc96")
    B, C, H, W = shape
    fused = run_case(base, "bc96")
    sch = EDMDPMSolverMultistepScheduler()
    sdata = 0.5
    ts = [float(torch.atan(sch.sigmas[0] / sdata)), float(torch.tensor(kw["intermediate_t"]))]
    win = torch.from_numpy(oeval.linear_weight_window(64).numpy()).cuda()
    starts = [0, 32]
    sample = torch.zeros(shape, device="cuda")
    cimg = cond.cuda()
    for k, t in enumerate(ts):
        z = noise[k].cuda()
        out = torch.zeros(shape, device="cuda")
        wsum = torch.zeros(shape, device="cuda")
        for ic, i0 in enumerate(starts):
            for jc, j0 in enumerate(starts):
                cv = process_latent_conditioning(cimg[..., ic:ic + 4, jc:jc + 4], kw["histogram_raw"],
                                                 kw["cond_means"], kw["cond_stds"], kw["noise_level"],
                                                 reference_sampler_nans=True)
                x_t = math.cos(t) * sample[..., i0:i0 + 64, j0:j0 + 64] + math.sin(t) * sdata * \
                    z[..., i0:i0 + 64, j0:j0 + 64]
                pred = -base(x_t / sdata, torch.full((B,), t, device="cuda"), [cv])
                s = math.cos(t) * x_t - math.sin(t) * sdata * pred
                out[..., i0:i0 + 64, j0:j0 + 64] += s * win
                wsum[..., i0:i0 + 64, j0:j0 + 64] += win
        sample = out / wsum
    err = rel_rms(fused, sample / sdata)
    print(f"\nfused vs public model: rel-RMS {err:.3e}")
    assert err <= 1e-2


# ------------------------------------------------------------------------------------------------ invariants
def test_tile_batch_is_a_free_choice_and_runs_replay_bitwise(base):
    ys = {tb: run_case(base, "bc96", tile_batch=tb) for tb in (1, 2, None)}
    for tb in (1, 2):
        assert rel_rms(ys[tb], ys[None]) <= 1e-2, tb
    check_golden(ys[1], "bc96")
    assert torch.equal(run_case(base, "bc96"), ys[None])
    a = run_case(base, "bc1", generator=torch.Generator().manual_seed(3))
    assert torch.equal(a, run_case(base, "bc1", generator=torch.Generator().manual_seed(3)))


def test_coarse_tile_batch_is_a_free_choice(coarse):
    cond_img = torch.randn(1, 5, 112, 112, generator=torch.Generator().manual_seed(8))
    snr = torch.tensor([[0.2, 0.5, 1.0, 0.5, 2.0]])

    def run(tb):
        torch.manual_seed(2)
        return sample_coarse_tiled(coarse, EDMDPMSolverMultistepScheduler(), cond_img, snr, steps=3, tile_size=64,
                                   tile_stride=48, generator=torch.Generator().manual_seed(9), tile_batch=tb)
    y1, y4 = run(1), run(None)
    assert rel_rms(y1, y4) <= 1e-2
    assert torch.equal(y4, run(None))


def test_evaluation_call_shape(base):
    """evaluation/base_consistency.py:175-187: 40 images, statistics and noise level on the device, a CUDA
    generator, tile 64, intermediate_t 0.61."""
    dev = torch.device("cuda")
    B = 40
    g = torch.Generator().manual_seed(12)
    cond = torch.randn(B, 7, 4, 4, generator=g).to(dev)
    hist = torch.randn(B, 5, generator=g).to(dev)
    y = sample_base_consistency(model=base, scheduler=EDMDPMSolverMultistepScheduler(), shape=(B, 5, 64, 64),
                                cond_inputs=cond, cond_means=torch.zeros(7, device=dev),
                                cond_stds=torch.ones(7, device=dev), noise_level=torch.zeros(B, 1, device=dev),
                                histogram_raw=hist, intermediate_t=0.61,
                                generator=torch.Generator(device=dev).manual_seed(1), tile_size=64)
    assert y.shape == (B, 5, 64, 64) and y.is_cuda
    assert bool(torch.isfinite(y).all()) and float(y.std()) > 0.05
