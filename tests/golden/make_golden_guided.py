"""Generate tests/golden/guided_golden.npz: two-model guided samplers of the UNMODIFIED reference (checkout at
$TERRAIN_DIFFUSION_REF), fp32 and the reference's own CPU bf16 autocast, on procedural weights (main seed 0, guide
seed 1; oracle.unet.procedural_state_dict re-creates them identically in the tests).

    python tests/golden/make_golden_guided.py

Cases (inputs are stored next to the outputs):
  base1   sample_base_diffusion untiled: BASE_CFG main + the same config at model_channels=128 as guide, B=2, 64^2,
          4 steps, guidance 2.15, 58-dim condition vectors given directly, noise from a seeded CPU generator
  base96  the same pair tiled over 96^2 (tile 64, stride 32: 2x2 tiles, 5x5 cond image), B=1
  dec     sample_decoder_diffusion_tiled on one 64^2 tile: DECODER_CFG main (seed 0) and guide (seed 1), 4 steps,
          guidance 1.5, score_scaling 1.2 (one tile: the shipped function does not reset its scheduler per tile)
<case>.ref_bf16_err is rel-RMS(bf16 autocast output, fp32 output) of the reference itself.
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
from terrain_diffusion.training.evaluation.sample_diffusion_base import sample_base_diffusion  # noqa: E402
from terrain_diffusion.training.evaluation.sample_diffusion_decoder import sample_decoder_diffusion_tiled  # noqa: E402

from oracle import unet as O  # noqa: E402
from tests.golden.make_golden import BASE_CFG  # noqa: E402

torch.set_grad_enabled(False)

GUIDE_CFG = dict(BASE_CFG, model_channels=128)
STEPS = 4
BASE_GUIDANCE = 2.15
DEC_GUIDANCE, DEC_SCORE_SCALING = 1.5, 1.2
NOISE_SEED = 7


def build_ref(cfg, seed):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(O.procedural_state_dict(cfg, seed=seed))
    return m


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def both(fn):
    """fp32 output and the reference's own bf16 autocast output of the same call."""
    t0 = time.time()
    y32 = fn().float()
    with torch.autocast("cpu", dtype=torch.bfloat16):
        y16 = fn().float()
    print(f"  {time.time() - t0:.0f}s  bf16 err {rel_rms(y16, y32):.4g}", flush=True)
    return y32, y16


def base_inputs():
    g = torch.Generator().manual_seed(11)
    cvec = torch.randn(2, 58, generator=g)
    cond_img = torch.randn(1, 7, 5, 5, generator=g)
    cond_img[:, 6] = 1.0                          # mask channel
    cond_img[0, 0, 2, 3] = float("nan")           # row 0: NaN -> cond_means[0] (sample_diffusion_base.py:36)
    means = np.array([0.3, -0.2, 10.0, 5.0, 800.0, 0.4, 0.5], dtype=np.float32)
    stds = np.array([1.5, 1.2, 8.0, 3.0, 600.0, 0.3, 0.5], dtype=np.float32)
    hist = torch.randn(1, 5, generator=g)
    noise_level = torch.tensor([[0.25]])
    return cvec, cond_img, means, stds, hist, noise_level


def main():
    out: dict = {}
    main_m, guide_m = build_ref(BASE_CFG, 0), build_ref(GUIDE_CFG, 1)
    cvec, cond_img, means, stds, hist, noise_level = base_inputs()
    out.update({"base.cvec": cvec.numpy(), "base.cond_img": cond_img.numpy(), "base.means": means,
                "base.stds": stds, "base.hist": hist.numpy(), "base.noise_level": noise_level.numpy(),
                "base.noise_seed": np.int64(NOISE_SEED), "base.steps": np.int64(STEPS),
                "base.guidance": np.float64(BASE_GUIDANCE)})

    def base1():
        sch = EDMDPMSolverMultistepScheduler()
        sch.set_timesteps(STEPS)
        return sample_base_diffusion(main_m, sch, (2, 5, 64, 64), [cvec], cond_means=means, cond_stds=stds,
                                     noise_level=noise_level, histogram_raw=hist, steps=STEPS, guide_model=guide_m,
                                     guidance_scale=BASE_GUIDANCE,
                                     generator=torch.Generator().manual_seed(NOISE_SEED))
    print("base1", flush=True)
    out["base1.y"], y16 = both(base1)
    out["base1.ref_bf16_err"] = np.float64(rel_rms(y16, out["base1.y"]))

    def base96():
        sch = EDMDPMSolverMultistepScheduler()
        sch.set_timesteps(STEPS)
        return sample_base_diffusion(main_m, sch, (1, 5, 96, 96), cond_img, cond_means=means, cond_stds=stds,
                                     noise_level=noise_level, histogram_raw=hist, steps=STEPS, guide_model=guide_m,
                                     guidance_scale=BASE_GUIDANCE,
                                     generator=torch.Generator().manual_seed(NOISE_SEED), tile_size=64)
    print("base96", flush=True)
    out["base96.y"], y16 = both(base96)
    out["base96.ref_bf16_err"] = np.float64(rel_rms(y16, out["base96.y"]))
    del main_m, guide_m

    dec_m, dec_g = build_ref(O.DECODER_CFG, 0), build_ref(O.DECODER_CFG, 1)
    g = torch.Generator().manual_seed(12)
    noise = torch.randn(1, 1, 64, 64, generator=g) * 80
    cond = torch.randn(1, 4, 64, 64, generator=g)
    out.update({"dec.noise": noise.numpy(), "dec.cond": cond.numpy(), "dec.steps": np.int64(STEPS),
                "dec.guidance": np.float64(DEC_GUIDANCE), "dec.score_scaling": np.float64(DEC_SCORE_SCALING)})

    def dec():
        return sample_decoder_diffusion_tiled(dec_m, EDMDPMSolverMultistepScheduler(), cond, noise, 64, 64,
                                              num_steps=STEPS, guidance_model=dec_g, guidance_scale=DEC_GUIDANCE,
                                              score_scaling=DEC_SCORE_SCALING)
    print("dec", flush=True)
    out["dec.y"], y16 = both(dec)
    out["dec.ref_bf16_err"] = np.float64(rel_rms(y16, out["dec.y"]))
    np.savez_compressed(HERE / "guided_golden.npz", **out)
    print(f"wrote {len(out)} arrays, {os.path.getsize(HERE / 'guided_golden.npz') / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
