"""T4/T5/T6/T7: the CUDA U-Net, scheduler, fused N-step solves and blend against the fp32 oracle and the golden
vectors recorded from the unmodified reference (tests/golden/reference_golden.npz).

Tolerance (SURVEY.md section 8c): bf16 tensor-core path vs the FP32 oracle -- rel-RMS <= 1.0e-2 per forward and per
N-step solve (the reference's own bf16-vs-fp32 deviation is 0.86 % / 0.98 %).  Integer / fp32 elementwise pieces
(scheduler step, blend) are held to fp32 round-off or bit-exactness as stated per test.
"""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import scheduler as osched
from oracle import tiling as otile
from oracle import unet as ounet
from terrain_diffusion_b200.inference import (BlendCanvas, DiffusionSolve, sample_decoder_consistency_tiled,
                                              sample_decoder_diffusion_tiled)
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "reference_golden.npz")
TOL = 1.0e-2


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def _gen_inputs(cfg, n, hw, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cfg["in_channels"], hw, hw, generator=g)
    t = torch.atan(torch.exp(torch.randn(n, generator=g) * 1.5) / 0.5)
    return x, t


@pytest.fixture(scope="module")
def decoder():
    cfg = ounet.DECODER_CFG
    sd = ounet.procedural_state_dict(cfg, seed=0)
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(sd)
    return m.cuda(), sd, cfg


def test_forward_matches_reference_golden_64(decoder):
    m, sd, cfg = decoder
    x, t = _gen_inputs(cfg, 1, 64, seed=1)
    y = m(x.cuda(), t.cuda(), []).cpu()
    ref = torch.from_numpy(G["decoder.y"])  # output of the UNMODIFIED reference, fp32 CPU
    assert float(ref.std()) > 0.5
    assert rel_rms(y, ref) < TOL


def test_forward_matches_reference_golden_128_batch2(decoder):
    m, sd, cfg = decoder
    x, t = _gen_inputs(cfg, 2, 128, seed=2)
    y = m(x.cuda(), t.cuda(), []).cpu()
    assert rel_rms(y, torch.from_numpy(G["decoder128.y"])) < TOL


def test_forward_256_matches_oracle(decoder):
    m, sd, cfg = decoder
    x, t = _gen_inputs(cfg, 1, 256, seed=7)
    ref = ounet.unet_forward(sd, cfg, x, t, [])
    y = m(x.cuda(), t.cuda(), []).cpu()
    assert rel_rms(y, ref) < TOL


def test_forward_graph_replay_is_deterministic_and_dtype_follows_input(decoder):
    m, sd, cfg = decoder
    x, t = _gen_inputs(cfg, 1, 64, seed=3)
    a = m(x.cuda(), t.cuda(), [])
    b = m(x.cuda(), t.cuda(), [])
    assert torch.equal(a, b)
    c = m(x.cuda().bfloat16(), t.cuda().bfloat16(), [])
    assert c.dtype == torch.bfloat16 and c.shape == (1, 1, 64, 64)


def test_forward_rejects_cpu_and_bad_sizes(decoder):
    from terrain_diffusion_b200._lib import TdxError
    m, sd, cfg = decoder
    with pytest.raises(TdxError):
        m(torch.zeros(1, 5, 64, 64), torch.zeros(1), [])
    with pytest.raises(ValueError):
        m(torch.zeros(1, 5, 72, 72, device="cuda"), torch.zeros(1, device="cuda"), [])


def test_coarse_model_with_float_conditioning_matches_reference_golden():
    cfg = dict(image_size=16, in_channels=11, out_channels=6, model_channels=128, model_channel_mults=[1],
               layers_per_block=2, attn_resolutions=[], midblock_attention=False, concat_balance=0.5,
               conditional_inputs=[["float", 64, 0.2]] * 5, fourier_scale="pos", block_kwargs={})
    sd = ounet.procedural_state_dict(cfg, seed=0)
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(sd)
    m = m.cuda()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 11, 64, 64, generator=g)
    t = torch.atan(torch.exp(torch.randn(1, generator=g) * 1.5) / 0.5)
    cond = [torch.randn(1, generator=g) for _ in range(5)]
    y = m(x.cuda(), t.cuda(), [c.cuda() for c in cond]).cpu()
    assert rel_rms(y, torch.from_numpy(G["coarse.y"])) < TOL


def test_base_latent_model_with_attention_matches_reference_golden():
    """SURVEY section 8f rank 1: the 253 M-parameter latent model (192..768 channels, tensor conditioning, one cosine
    self-attention block at 8x8 tokens) vs the unmodified reference's fp32 output."""
    cfg = dict(image_size=512, in_channels=5, out_channels=5, model_channels=192, model_channel_mults=[1, 2, 3, 4],
               layers_per_block=3, attn_resolutions=[8, 16], midblock_attention=True, concat_balance=0.5,
               conditional_inputs=[["tensor", 58, 1.0]], fourier_scale="pos", block_kwargs={"dropout": 0.1})
    sd = ounet.procedural_state_dict(cfg, seed=0)
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(sd)
    del sd
    m = m.cuda()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 5, 64, 64, generator=g)
    t = torch.atan(torch.exp(torch.randn(1, generator=g) * 1.5) / 0.5)
    cond = [torch.randn(1, 58, generator=g)]
    y = m(x.cuda(), t.cuda(), [c.cuda() for c in cond]).cpu()
    ref = torch.from_numpy(G["base.y"])
    assert float(ref.std()) > 0.5
    assert rel_rms(y, ref) < TOL
    # batch of 4 tiles (the product's latent stage batches up to 16): rows must agree with the single-tile result
    y4 = m(x.cuda().repeat(4, 1, 1, 1), t.cuda().repeat(4), [cond[0].cuda().repeat(4, 1)]).cpu()
    assert rel_rms(y4[2:3], ref) < TOL


# ------------------------------------------------------------------------------------------------ scheduler
@pytest.mark.parametrize("n", [4, 12, 20])
def test_scheduler_step_sequence_matches_reference_golden(n):
    s = EDMDPMSolverMultistepScheduler()
    s.set_timesteps(n)
    np.testing.assert_array_equal(s.sigmas.numpy(), G[f"sched{n}.sigmas"])
    np.testing.assert_array_equal(s.timesteps.numpy(), G[f"sched{n}.timesteps"])
    traj = torch.from_numpy(G[f"sched{n}.traj"])
    g = torch.Generator().manual_seed(100 + n)
    x = (torch.randn(1, 1, 8, 8, generator=g) * 80).cuda()
    for i, (t, sigma) in enumerate(zip(s.timesteps, s.sigmas)):
        f = torch.randn(1, 1, 8, 8, generator=g).cuda()
        x = s.step(f, t, x).prev_sample
        ref = traj[2 * i + 1, 0]
        # fp32 closed form vs the reference's fp32 log/exp form: <= 1e-6 of the sample magnitude
        assert float((x.cpu() - ref).abs().max()) <= 1e-6 * max(1.0, float(ref.abs().max())) * 8, (n, i)


def test_scheduler_requires_set_timesteps_and_cuda():
    from terrain_diffusion_b200._lib import TdxError
    s = EDMDPMSolverMultistepScheduler()
    with pytest.raises(ValueError):
        s.step(torch.zeros(1, device="cuda"), torch.tensor(0.0), torch.zeros(1, device="cuda"))
    s.set_timesteps(4)
    with pytest.raises(TdxError):
        s.step(torch.zeros(1), s.timesteps[0], torch.zeros(1))


# ------------------------------------------------------------------------------------------------ N-step solves
def test_cfg1_single_tile_4_step_matches_reference_golden(decoder):
    """BASELINE configs[0] on the GPU path vs the unmodified reference's fp32 CPU result."""
    m, sd, cfg = decoder
    g = torch.Generator().manual_seed(1)
    noise = torch.randn(1, 1, 64, 64, generator=g) * 80
    cond = torch.randn(1, 4, 64, 64, generator=g)
    y = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond.cuda(), noise.cuda(), 64, 64,
                                       num_steps=4).cpu()
    assert rel_rms(y, torch.from_numpy(G["cfg1.y"])) < TOL


def test_fused_solve_equals_unfused_model_plus_scheduler(decoder):
    """The one-graph solve (scale folded into conv_in, scheduler.step folded into conv_out) == calling the public
    model + scheduler.step per step."""
    m, sd, cfg = decoder
    g = torch.Generator().manual_seed(9)
    noise = (torch.randn(2, 1, 64, 64, generator=g) * 80).cuda()
    cond = torch.randn(2, 4, 64, 64, generator=g).cuda()
    sch = EDMDPMSolverMultistepScheduler()
    fused = DiffusionSolve(m, sch, 2, 64, 64, 6).run(noise, cond).clone()
    sch.set_timesteps(6)
    x = noise.clone()
    for t, sigma in zip(sch.timesteps, sch.sigmas):
        mo = m(torch.cat([sch.precondition_inputs(x, sigma), cond], dim=1),
               sch.trigflow_precondition_noise(sigma.view(-1).expand(2)).cuda(), [])
        x = sch.step(mo, t, x).prev_sample
    assert rel_rms(fused, x) < 2e-3


def test_cfg2_one_256_tile_20_steps_matches_oracle(decoder):
    """BASELINE configs[1]: 20-step solve of one 256x256 tile vs the fp32 oracle solve."""
    m, sd, cfg = decoder
    g = torch.Generator().manual_seed(1)
    noise = torch.randn(1, 1, 256, 256, generator=g) * 80
    cond = torch.randn(1, 4, 256, 256, generator=g)
    ref = otile.sample_decoder_diffusion_tiled(lambda x, t: ounet.unet_forward(sd, cfg, x, t, []),
                                               osched.OracleScheduler, cond, noise, 256, 256, num_steps=20)
    y = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond.cuda(), noise.cuda(), 256, 256,
                                       num_steps=20).cpu()
    assert rel_rms(y, ref) < TOL


def test_multi_tile_diffusion_blend_matches_oracle_and_batching_is_bit_identical(decoder):
    m, sd, cfg = decoder
    g = torch.Generator().manual_seed(4)
    noise = torch.randn(1, 1, 96, 96, generator=g) * 80
    cond = torch.randn(1, 4, 96, 96, generator=g)
    ref = otile.sample_decoder_diffusion_tiled(lambda x, t: ounet.unet_forward(sd, cfg, x, t, []),
                                               osched.OracleScheduler, cond, noise, 64, 32, num_steps=4)
    a = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond.cuda(), noise.cuda(), 64, 32,
                                       num_steps=4, tile_batch=1)
    b = sample_decoder_diffusion_tiled(m, EDMDPMSolverMultistepScheduler(), cond.cuda(), noise.cuda(), 64, 32,
                                       num_steps=4, tile_batch=4)
    assert rel_rms(a.cpu(), ref) < TOL
    assert rel_rms(b.cpu(), ref) < TOL


def test_consistency_multi_tile_matches_reference_golden(decoder):
    m, sd, cfg = decoder
    g = torch.Generator().manual_seed(5)
    noise = torch.randn(1, 1, 96, 96, generator=g)
    cond = torch.randn(1, 4, 96, 96, generator=g)
    y = sample_decoder_consistency_tiled(m, EDMDPMSolverMultistepScheduler(), cond.cuda(), noise.cuda(), 64, 32,
                                         intermediate_t=[0.6]).cpu()
    assert rel_rms(y, torch.from_numpy(G["consistency96.y"])) < TOL


# ------------------------------------------------------------------------------------------------ blend
def test_blend_canvas_is_bit_exact_with_oracle():
    """One image, and a batch of b images on one canvas of b * C planes sharing one weight sum, as the tiled samplers
    blend it."""
    for b in (1, 3):
        g = torch.Generator().manual_seed(12)
        h, w, t, stride, c = 100, 148, 64, 48, 3
        val = torch.zeros(b, c, h, w)
        ws = torch.zeros(b, 1, h, w)
        win = otile.linear_weight_window(t)
        cv = BlendCanvas(b * c, h, w, "cuda")
        for i0 in otile.tile_starts(h, t, stride):
            for j0 in otile.tile_starts(w, t, stride):
                tile = torch.randn(b, c, t, t, generator=g)
                otile.accumulate(val, ws, tile, win[None, None], i0, j0)
                cv.accumulate(tile.reshape(b * c, t, t).cuda(), i0, j0)
        assert torch.equal(cv.val.cpu(), val.reshape(b * c, h, w)), b
        assert torch.equal(cv.wsum.cpu(), ws[0, 0]), b
        assert torch.equal(cv.normalized().cpu().view(b, c, h, w), val / ws), b
        assert torch.equal(cv.normalized(0.5).cpu().view(b, c, h, w), val / ws / 0.5), b
        assert torch.equal(cv.packed().cpu(), torch.cat([val.reshape(b * c, h, w), ws[0]], dim=0)), b


def test_blend_canvas_negative_world_coordinates_and_clipping():
    cv = BlendCanvas(1, 32, 32, "cuda", origin=(-16, -16))
    tile = torch.ones(1, 16, 16, device="cuda")
    cv.accumulate(tile, -24, -24)  # only the lower-right 8x8 quadrant lands on the canvas
    win = otile.linear_weight_window(16)
    assert torch.equal(cv.wsum.cpu()[:8, :8], win[8:, 8:])
    assert float(cv.wsum.cpu()[8:, :].abs().sum()) == 0.0
