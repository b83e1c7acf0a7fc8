"""Golden vectors for the pooled coarse stage (`coarse_pooling`), produced by the reference's OWN method bodies.

`extract()` of make_golden_stages.py compiles the reference's `_coarse_inference`, `_pool_coarse_conditioning` and
`_pool_channel` unchanged; they are called with a small stand-in for `self` (world_pipeline.py:909-1016).

  epilogue cases  `_coarse_inference` with its solve replaced by a stand-in scheduler whose one step returns a given raw
                  sample (tests/_coarse_pool_inputs.py: NaN, +-inf, +-0, ties), so everything after the solve --
                  de-normalisation, the channel-1 difference, pooling and the packed output -- is the reference's code,
                  for every pool size and (elev, p5) mode pair, plus two mode strings the reference does not name.
                  Channels 2-6 (average-pooled data and weights) do not depend on the modes and are stored once per
                  pool size (`epi_n{n}_rest`); channels 0-1 per mode pair (`epi_n{n}_{elev}_{p5}`).  At n = 1 the modes
                  are unused, so only `epi_n1_avg_avg` is stored.
  stage cases     `_coarse_inference(..., pool_size=n)`, the full 20-step solve with the procedural coarse weights, at
                  window (0, 1, -2) for (2, max, min), (4, avg, avg) and (16, min, max) (`stage_n{n}_{elev}_{p5}`).

    TERRAIN_DIFFUSION_REF=<reference checkout> python tests/golden/make_golden_coarse_pool.py
"""
from __future__ import annotations

import functools
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

from make_golden_stages import build, extract  # noqa: E402  (sets up the reference import paths)

from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler  # noqa: E402
from tests._coarse_pool_inputs import (MODES, POOL_SIZES, SIGMA_DATA, STAGE_CASES, STAGE_CTX,  # noqa: E402
                                       UNKNOWN_MODES, epilogue_input)
from tests._stage_inputs import SEED, stage_inputs  # noqa: E402
from tests.test_oracle_golden import COARSE_CFG  # noqa: E402

torch.set_grad_enabled(False)


class GivenSample:
    """Scheduler and model for `_coarse_inference` whose one-step 'solve' ends in a given raw sample."""

    def __init__(self, raw):
        self.raw = raw
        self.config = SimpleNamespace(sigma_data=SIGMA_DATA)
        self.timesteps, self.sigmas = torch.zeros(1), torch.ones(1)

    def set_timesteps(self, n):
        pass

    def precondition_inputs(self, sample, sigma):
        return sample

    def trigflow_precondition_noise(self, sigma):
        return sigma

    def step(self, model_out, t, sample):
        return SimpleNamespace(prev_sample=self.raw[None].clone())

    def model(self, x, noise_labels=None, conditional_inputs=None):
        return x[:, :6]


def stand_in(ns, model, means, stds, elev_mode, p5_mode, cond_map):
    fake = SimpleNamespace(device=torch.device("cpu"), _dtype=None, seed=SEED, coarse_model=model, log_mode="quiet",
                           kwargs={"coarse_means": [float(v) for v in means], "coarse_stds": [float(v) for v in stds],
                                   "elev_coarse_pool_mode": elev_mode, "p5_coarse_pool_mode": p5_mode},
                           _conditioning_model_input=lambda i1, i2, j1, j2: cond_map.clone())
    fake._pool_channel = functools.partial(ns["_pool_channel"], fake)
    fake._pool_coarse_conditioning = functools.partial(ns["_pool_coarse_conditioning"], fake)
    return fake


def main():
    ns = extract()
    out = {}
    inp = stage_inputs()
    t_cond = torch.atan(inp["cond_snr"])
    cond_inputs = [v.detach().view(-1) for v in torch.log(torch.tan(t_cond) / 8.0)]

    # ---------------- epilogue cases: the reference's code after the solve, on a given raw sample
    x, means, stds = epilogue_input()
    given = GivenSample(x)
    for n in POOL_SIZES:
        ww = ns["linear_weight_window"](64 // n, "cpu", torch.float32)
        pairs = [("avg", "avg")] if n == 1 else [(e, p) for e in MODES for p in MODES] + [UNKNOWN_MODES]
        rest = None
        for e, p in pairs:
            fake = stand_in(ns, given.model, means, stds, e, p, inp["coarse_map"])
            got = ns["_coarse_inference"](fake, (0, 0, 0), given, ww, t_cond, cond_inputs, pool_size=n).numpy()
            assert got.shape == (7, 64 // n, 64 // n), got.shape
            if rest is None:
                rest = got[2:]
            assert rest.tobytes() == got[2:].tobytes(), (n, e, p)       # channels 2-6 do not depend on the modes
            out[f"epi_n{n}_{e}_{p}"] = got[:2]
        out[f"epi_n{n}_rest"] = rest
    out["epi_means"], out["epi_stds"] = means.numpy(), stds.numpy()

    # ---------------- stage cases: the full 20-step solve, pooled
    coarse = build(COARSE_CFG)
    for n, e, p in STAGE_CASES:
        fake = stand_in(ns, coarse, inp["coarse_means"], inp["coarse_stds"], e, p, inp["coarse_map"])
        ww = ns["linear_weight_window"](64 // n, "cpu", torch.float32)
        sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
        out[f"stage_n{n}_{e}_{p}"] = ns["_coarse_inference"](fake, STAGE_CTX, sched, ww, t_cond, cond_inputs,
                                                             pool_size=n).numpy()
    out["torch_version"] = np.asarray(torch.__version__)
    out["cpu_capability"] = np.asarray(torch.backends.cpu.get_cpu_capability())
    np.savez_compressed(HERE / "coarse_pool_golden.npz", **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
