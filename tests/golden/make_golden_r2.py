"""Round-2 golden fixtures (tests/golden/parity_r2_golden.npz), generated in the build container from the UNMODIFIED
reference (checkout at $TERRAIN_DIFFUSION_REF; the GPU tests only read the stored result):

  ref_bf16_err_{64,128,256}   rel-RMS of the reference's OWN bf16 mode (model.to(bfloat16), bf16 input -- what
                              WorldPipeline does for dtype='bf16', world_pipeline.py:414-419) against its fp32 output on
                              the inputs of tests/test_unet_gpu.py: the second half of the SURVEY 8(c) tolerance
                              ("<= 1.25 x the reference's own bf16-vs-fp32 error on the same inputs").
  fwd512_sub4                 reference fp32 forward of the decoder at 512 x 512 (the product tile), every 4th pixel.
  cfg3_sub8                   BASELINE config 3 geometry: 1664^2 canvas, tile 512 / stride 384 (4 x 4 = 16 tiles,
                              training/evaluation/__init__.py:16-22), 2 solver steps per tile with a per-tile scheduler
                              reset (sample_diffusion_base.py:147), blended; reference model + reference scheduler + the
                              reference's tile helpers in the loop shape of sample_diffusion_decoder.py:91-125; every 8th
                              pixel.
Inputs are torch.Generator streams (seeds below) so the tests re-create them bit for bit.

    python tests/golden/make_golden_r2.py
"""
from __future__ import annotations

import os

import sys
import time
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]

from terrain_diffusion.models.edm_unet import EDMUnet2D  # noqa: E402
from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler  # noqa: E402
from terrain_diffusion.training.evaluation import _linear_weight_window, _tile_starts  # noqa: E402

from oracle import unet as O  # noqa: E402

torch.set_grad_enabled(False)


def rel_rms(a, b):
    return float((a.float() - b.float()).square().mean().sqrt() / b.float().square().mean().sqrt())


def gen_inputs(cfg, n, hw, seed):
    """Same stream as tests/test_unet_gpu.py::_gen_inputs."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cfg["in_channels"], hw, hw, generator=g)
    t = torch.atan(torch.exp(torch.randn(n, generator=g) * 1.5) / 0.5)
    return x, t


def cfg3_inputs(size=1664, seed=21):
    g = torch.Generator().manual_seed(seed)
    noise = torch.randn(1, 1, size, size, generator=g)
    cond = torch.randn(1, 4, size, size, generator=g)
    return noise, cond


def main():
    cfg = O.DECODER_CFG
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(O.procedural_state_dict(cfg, seed=0))
    out = {}
    # ---- the reference's own bf16 deviation
    mb = EDMUnet2D(**cfg).eval()
    mb.load_state_dict(O.procedural_state_dict(cfg, seed=0))
    mb = mb.to(torch.bfloat16)
    for n, hw, seed in ((1, 64, 1), (2, 128, 2), (1, 256, 7)):
        x, t = gen_inputs(cfg, n, hw, seed)
        t0 = time.time()
        y32 = m(x, t, [])
        yb = mb(x.bfloat16(), t.bfloat16(), [])
        out[f"ref_bf16_err_{hw}"] = np.float64(rel_rms(yb, y32))
        print(hw, out[f"ref_bf16_err_{hw}"], f"{time.time() - t0:.1f}s", flush=True)
    del mb
    # ---- 512 x 512 forward
    x, t = gen_inputs(cfg, 1, 512, 11)
    out["fwd512_sub4"] = m(x, t, [])[:, :, ::4, ::4].contiguous().numpy()
    print("fwd512 done", flush=True)
    # ---- config 3 geometry, 2 steps per tile
    noise, cond = cfg3_inputs()
    tile, stride, steps = 512, 384, 2
    sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
    sched.set_timesteps(steps)
    noise = noise * sched.sigmas[0]
    weights = _linear_weight_window(tile, "cpu", torch.float32)          # [1, 1, T, T]
    acc = torch.zeros_like(noise)
    acc_w = torch.zeros_like(noise)
    starts = _tile_starts(noise.shape[-1], tile, stride)
    assert starts == [0, 384, 768, 1152], starts
    for i0 in starts:
        for j0 in starts:
            sched.set_timesteps(steps)          # per-tile reset of the stateful scheduler
            samples = noise[..., i0:i0 + tile, j0:j0 + tile]
            tc = cond[..., i0:i0 + tile, j0:j0 + tile]
            for tt, sigma in zip(sched.timesteps, sched.sigmas):
                scaled = sched.precondition_inputs(samples, sigma)
                cnoise = sched.trigflow_precondition_noise(sigma.view(-1))
                mo = m(torch.cat([scaled, tc], dim=1), noise_labels=cnoise, conditional_inputs=[])
                samples = sched.step(mo, tt, samples).prev_sample
            acc[..., i0:i0 + tile, j0:j0 + tile] += samples * weights
            acc_w[..., i0:i0 + tile, j0:j0 + tile] += weights
            print("tile", i0, j0, flush=True)
    res = acc / acc_w
    out["cfg3_sub8"] = res[:, :, ::8, ::8].contiguous().numpy()
    out["cfg3_starts"] = np.asarray(starts, dtype=np.int64)
    np.savez_compressed(HERE / "parity_r2_golden.npz", **out)
    print({k: (getattr(v, "shape", ()), float(np.abs(v).mean())) for k, v in out.items()})


if __name__ == "__main__":
    main()
