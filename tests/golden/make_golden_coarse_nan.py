"""Golden vectors for a coarse window whose conditioning has NaN cells, produced by the reference's OWN
`_coarse_inference` (through `extract()` of make_golden_stages.py, world_pipeline.py:909-959).

The reference feeds `_conditioning_model_input` -- imported rasters copied under their mask, or a user
`conditioning_fn` -- into the coarse solve without filtering NaN (its latent stage `nan_to_num`s the result later), so a
nodata cell spreads through the window's 20-step solve.  Recorded: the window (0, 1, -2) of tests/_stage_inputs.py with
the NaN cells of tests/_nonfinite.coarse_nan_map, the procedural coarse weights, CPU fp32.  oneDNN is switched off so
that the convolutions are torch's direct im2col + GEMM path: oneDNN may pick Winograd for a 3x3, which spreads a NaN
over a whole transform tile -- an artefact of that algorithm, not of the model.  Stored: `nan` (the packed [7, 64, 64]
output) and, as a check of the recording, `clean` (the same window without the NaN cells).

    TERRAIN_DIFFUSION_REF=<reference checkout> python tests/golden/make_golden_coarse_nan.py
"""
from __future__ import annotations

import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

from make_golden_stages import build, extract  # noqa: E402  (sets up the reference import paths)

from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler  # noqa: E402
from tests._nonfinite import COARSE_NAN_CTX, coarse_nan_map  # noqa: E402
from tests._stage_inputs import SEED, stage_inputs  # noqa: E402
from tests.test_oracle_golden import COARSE_CFG  # noqa: E402

torch.set_grad_enabled(False)
torch.backends.mkldnn.enabled = False


def main():
    ns = extract()
    inp = stage_inputs()
    t_cond = torch.atan(inp["cond_snr"])
    cond_inputs = [v.detach().view(-1) for v in torch.log(torch.tan(t_cond) / 8.0)]
    coarse = build(COARSE_CFG)
    ww = ns["linear_weight_window"](64, "cpu", torch.float32)
    out = {}
    for name, cmap in (("nan", coarse_nan_map(inp["coarse_map"])), ("clean", inp["coarse_map"])):
        fake = SimpleNamespace(device=torch.device("cpu"), _dtype=None, seed=SEED, coarse_model=coarse,
                               log_mode="quiet",
                               kwargs={"coarse_means": inp["coarse_means"].tolist(),
                                       "coarse_stds": inp["coarse_stds"].tolist()},
                               _conditioning_model_input=lambda i1, i2, j1, j2, m=cmap: m.clone())
        sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
        out[name] = ns["_coarse_inference"](fake, COARSE_NAN_CTX, sched, ww, t_cond, cond_inputs).numpy()
    out["torch_version"] = np.asarray(torch.__version__)
    np.savez_compressed(HERE / "coarse_nan_golden.npz", **out)
    print({k: (v.shape, int(np.isnan(v).sum())) for k, v in out.items() if v.dtype != np.dtype("<U0")
           and v.dtype.kind == "f"})


if __name__ == "__main__":
    main()
