"""Golden vectors for the phase split of the multi-phase sampler: the reference's OWN `build_timestep_ranges`
(annotated_infinite_panorama.py:84-102; the file imports diffusers / infinite_tensor, so the function is extracted with
ast and compiled unchanged) on the demo's DDIM-style timesteps and on an EDM-scheduler timestep table.

    python tests/golden/make_golden_phases.py     ->  tests/golden/phases_golden.npz
"""
import os
import ast
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]
from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler  # noqa: E402


def main():
    tree = ast.parse((REF / "annotated_infinite_panorama.py").read_text())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "build_timestep_ranges"]
    ns = {"torch": torch}
    exec(compile(ast.Module(body=fn, type_ignores=[]), "panorama_extract", "exec"), ns)
    btr = ns["build_timestep_ranges"]
    out = {}
    # the demo's configuration: 50 DDIM-style steps over 1000 training timesteps, thresholds (400, 600, 750, 900)
    ts = torch.arange(0, 1000, 20).flip(0) + 1
    cases = {"demo": (ts, (400, 600, 750, 900)), "unsorted": (ts, (750, 400)), "none": (ts, ()),
             "empty_phase": (ts, (2000, 500))}
    s = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
    s.set_timesteps(12)
    cases["edm12"] = (s.timesteps, (0.25 * np.log(5.0), 0.25 * np.log(0.3)))
    out["edm12_timesteps"] = s.timesteps.numpy()
    for name, (t, th) in cases.items():
        r = btr(t, th)
        out[f"{name}.lens"] = np.asarray([len(x) for x in r], dtype=np.int64)
        out[f"{name}.concat"] = torch.cat([x.float() for x in r]).numpy()
        out[f"{name}.thresholds"] = np.asarray(th, dtype=np.float64)
    out["demo.timesteps"] = ts.numpy()
    np.savez_compressed(HERE / "phases_golden.npz", **out)
    print({k: v.tolist() for k, v in out.items() if k.endswith(".lens")})


if __name__ == "__main__":
    main()
