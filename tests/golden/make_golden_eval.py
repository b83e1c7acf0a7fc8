"""Generate tests/golden/eval_golden.npz: the consistency-base and coarse evaluation samplers of the UNMODIFIED
reference (checkout at $TERRAIN_DIFFUSION_REF), fp32 and the reference's own CPU bf16 autocast, on procedural weights
(oracle.unet.procedural_state_dict, seed 0, re-created identically in the tests).

    python tests/golden/make_golden_eval.py

Cases (inputs are stored next to the outputs):
  bc1      sample_base_consistency, BASE_CFG, B=2, 64^2, one tile, 4x4 cond image with a NaN in row 0's elevation
           channel, intermediate_t 0.61, noise from a seeded CPU generator
  bc96     the same over 96^2 (tile 64, stride 32: 2x2 tiles, 5x5 cond image), B=1, explicit noise=[z0, z1]
  coarse1  sample_coarse_tiled, COARSE_CFG, B=1, one 64^2 tile, 4 steps, cond_snr [1, 5]; the conditioning noise
           comes from the seeded global CPU generator, the tile noise from a seeded CPU generator (one tile: the
           shipped function does not reset its scheduler per tile; B=1: with B > 1 its [1]-shaped float
           conditions fail to stack against the [B]-row noise embedding in mp_sum)
<case>.ref_bf16_err is rel-RMS(bf16 output, fp32 output) of the reference itself.  The coarse sampler wraps its model
call in torch.autocast(dtype=dtype); CPU autocast cannot target fp32 and disables itself, which switches an outer bf16
autocast off.  Its bf16 run therefore hands it the same model behind a wrapper that enters CPU bf16 autocast around
each forward, so that, as in the other cases, the model computes in bf16 and the sampler in fp32.  (The call with
dtype=torch.bfloat16 is no alternative: its bf16 blend window rounds 1 - 0.999 to 0 on the tile border and divides 0 by
0 there.)
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
from terrain_diffusion.training.evaluation.sample_coarse import sample_coarse_tiled  # noqa: E402
from terrain_diffusion.training.evaluation.sample_diffusion_base import sample_base_consistency  # noqa: E402

from oracle import unet as O  # noqa: E402
from tests.golden.make_golden import BASE_CFG, COARSE_CFG  # noqa: E402

torch.set_grad_enabled(False)

INTERMEDIATE_T = 0.61
NOISE_SEED = 7
COARSE_STEPS = 4
COND_SEED, TILE_SEED = 13, 17


def build_ref(cfg, seed):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(O.procedural_state_dict(cfg, seed=seed))
    return m


class Bf16Forward(torch.nn.Module):
    """`model` with every forward under CPU bf16 autocast (the coarse sampler's own autocast would switch it off)."""

    def __init__(self, model):
        super().__init__()
        self.model = model
        self.config = model.config

    def forward(self, *args, **kwargs):
        with torch.autocast("cpu", dtype=torch.bfloat16):
            return self.model(*args, **kwargs)


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def both(fn, fn16=None):
    """fp32 output and the reference's own bf16 output of the same call (CPU bf16 autocast)."""
    t0 = time.time()
    y32 = fn().float()
    with torch.autocast("cpu", dtype=torch.bfloat16):
        y16 = (fn16 or fn)().float()
    print(f"  {time.time() - t0:.0f}s  bf16 err {rel_rms(y16, y32):.4g}", flush=True)
    return y32, y16


def base_inputs():
    g = torch.Generator().manual_seed(11)
    means = np.array([0.3, -0.2, 10.0, 5.0, 800.0, 0.4, 0.5], dtype=np.float32)
    stds = np.array([1.5, 1.2, 8.0, 3.0, 600.0, 0.3, 0.5], dtype=np.float32)
    cond4 = torch.randn(2, 7, 4, 4, generator=g) * torch.from_numpy(stds).view(1, -1, 1, 1) + \
        torch.from_numpy(means).view(1, -1, 1, 1)
    cond4[:, 6] = 1.0                              # mask channel
    cond4[0, 0, 1, 2] = float("nan")               # row 0: NaN -> cond_means[0] (sample_diffusion_base.py:36)
    cond5 = torch.randn(1, 7, 5, 5, generator=g) * torch.from_numpy(stds).view(1, -1, 1, 1) + \
        torch.from_numpy(means).view(1, -1, 1, 1)
    cond5[:, 6] = 1.0
    hist1 = torch.randn(2, 5, generator=g)
    hist96 = torch.randn(1, 5, generator=g)
    z96 = torch.randn(2, 1, 5, 96, 96, generator=g)
    return means, stds, cond4, cond5, hist1, hist96, z96


def main():
    out: dict = {}
    base = build_ref(BASE_CFG, 0)
    means, stds, cond4, cond5, hist1, hist96, z96 = base_inputs()
    out.update({"bc.means": means, "bc.stds": stds, "bc.intermediate_t": np.float64(INTERMEDIATE_T),
                "bc1.cond_img": cond4.numpy(), "bc1.hist": hist1.numpy(), "bc1.noise_level": np.zeros((2, 1), np.float32),
                "bc1.noise_seed": np.int64(NOISE_SEED), "bc96.cond_img": cond5.numpy(), "bc96.hist": hist96.numpy(),
                "bc96.noise_level": np.full((1, 1), 0.25, np.float32), "bc96.noise": z96.numpy()})

    def bc1():
        return sample_base_consistency(base, EDMDPMSolverMultistepScheduler(), (2, 5, 64, 64), cond4.clone(),
                                       cond_means=means, cond_stds=stds, noise_level=torch.zeros(2, 1),
                                       histogram_raw=hist1, intermediate_t=INTERMEDIATE_T,
                                       generator=torch.Generator().manual_seed(NOISE_SEED), tile_size=64)
    print("bc1", flush=True)
    y32, y16 = both(bc1)
    out["bc1.y"], out["bc1.ref_bf16_err"] = y32.numpy(), np.float64(rel_rms(y16, y32))

    def bc96():
        return sample_base_consistency(base, EDMDPMSolverMultistepScheduler(), (1, 5, 96, 96), cond5.clone(),
                                       cond_means=means, cond_stds=stds, noise_level=torch.full((1, 1), 0.25),
                                       histogram_raw=hist96, intermediate_t=INTERMEDIATE_T, tile_size=64,
                                       noise=[z96[0], z96[1]])
    print("bc96", flush=True)
    y32, y16 = both(bc96)
    out["bc96.y"], out["bc96.ref_bf16_err"] = y32.numpy(), np.float64(rel_rms(y16, y32))
    del base

    coarse = build_ref(COARSE_CFG, 0)
    g = torch.Generator().manual_seed(12)
    cond_img = torch.randn(1, 5, 64, 64, generator=g)
    cond_snr = torch.tensor([[0.1, 0.5, 0.5, 0.5, 0.5]])
    out.update({"coarse1.cond_img": cond_img.numpy(), "coarse1.cond_snr": cond_snr.numpy(),
                "coarse1.steps": np.int64(COARSE_STEPS), "coarse1.cond_seed": np.int64(COND_SEED),
                "coarse1.tile_seed": np.int64(TILE_SEED)})

    def coarse1(model=coarse):
        torch.manual_seed(COND_SEED)
        return sample_coarse_tiled(model, EDMDPMSolverMultistepScheduler(), cond_img.clone(), cond_snr,
                                   steps=COARSE_STEPS, generator=torch.Generator().manual_seed(TILE_SEED))
    print("coarse1", flush=True)
    y32, y16 = both(coarse1, lambda: coarse1(Bf16Forward(coarse)))
    out["coarse1.y"], out["coarse1.ref_bf16_err"] = y32.numpy(), np.float64(rel_rms(y16, y32))
    np.savez_compressed(HERE / "eval_golden.npz", **out)
    print(f"wrote {len(out)} arrays, {os.path.getsize(HERE / 'eval_golden.npz') / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
