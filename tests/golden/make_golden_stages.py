"""Golden vectors for the three pipeline stage callbacks, produced by the reference's OWN method bodies.

`terrain_diffusion/inference/world_pipeline.py` cannot be imported here (it needs infinite_tensor, h5py, rasterio, ...),
so the method definitions of WorldPipeline._decoder_inference / _latent_inference / _coarse_inference (+ the helpers
they call) are extracted from the reference source with `ast` at run time, compiled unchanged, and called with a small
stand-in for `self` that carries exactly the attributes they read.  Models are the reference's EDMUnet2D on CPU fp32
with procedural weights.  Nothing from the reference is copied into the repo; only inputs seeds and outputs are stored
(tests/golden/stages_golden.npz).

    python tests/golden/make_golden_stages.py
"""
from __future__ import annotations

import os

import ast
import functools
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]

from terrain_diffusion.inference import portable_rng as ref_rng  # noqa: E402
from terrain_diffusion.models.edm_unet import EDMUnet2D  # noqa: E402
from terrain_diffusion.models.mp_layers import mp_concat  # noqa: E402
from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler  # noqa: E402

from oracle import unet as O  # noqa: E402
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG  # noqa: E402
from tests._stage_inputs import SEED, stage_inputs  # noqa: E402

torch.set_grad_enabled(False)


def extract():
    src = (REF / "terrain_diffusion/inference/world_pipeline.py").read_text()
    tree = ast.parse(src)
    want_fn = {"_tile_seed", "gaussian_noise_patch", "linear_weight_window"}
    want_m = {"_decoder_inference", "_latent_inference", "_coarse_inference", "_process_latent_conditioning",
              "_pool_coarse_conditioning", "_pool_channel", "_get_padded_batch_size"}
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in want_fn]
    for n in tree.body:
        if isinstance(n, ast.ClassDef) and n.name == "WorldPipeline":
            body += [m for m in n.body if isinstance(m, ast.FunctionDef) and m.name in want_m]
    ns = {"np": np, "torch": torch, "fill_standard_normal": ref_rng.fill_standard_normal,
          "standard_normal": ref_rng.standard_normal, "mp_concat": mp_concat, "MOCK": False}
    exec(compile(ast.Module(body=body, type_ignores=[]), "world_pipeline_extract", "exec"), ns)
    return ns


def latent_seed_offsets():
    """The seed_offset constants of the reference's _build_latent_stage call sites (world_pipeline.py:1133-1203):
    [init phase, first T_INTER phase] -- read from the source so the pipeline's wiring is pinned, not assumed."""
    src = (REF / "terrain_diffusion/inference/world_pipeline.py").read_text()
    vals = set()
    for n in ast.walk(ast.parse(src)):
        if isinstance(n, ast.FunctionDef) and n.name == "_build_latent_stage":
            for kw in (k for c in ast.walk(n) if isinstance(c, ast.Call) for k in c.keywords):
                if kw.arg != "seed_offset":
                    continue
                v = kw.value
                if isinstance(v, ast.Constant):
                    vals.add(int(v.value))
                elif isinstance(v, ast.BinOp) and isinstance(v.left, ast.Constant):   # 5820 + i
                    vals.add(int(v.left.value))
    return sorted(vals)


def build(cfg):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(O.procedural_state_dict(cfg, seed=0))
    return m


def main():
    ns = extract()
    out = {}
    offs = latent_seed_offsets()
    assert len(offs) == 2, offs
    out["latent_seed_offsets"] = np.asarray(offs, dtype=np.int64)
    inp = stage_inputs()
    sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)

    # ---------------- decoder stage: tile 128 / stride 96, window index with a negative coordinate, 1 and 2 steps
    dec = build(O.DECODER_CFG)
    fake = SimpleNamespace(device=torch.device("cpu"), _dtype=None, latent_compression=8, seed=SEED, decoder_model=dec,
                           log_mode="quiet")
    ww = ns["linear_weight_window"](128, "cpu", torch.float32)
    t0 = torch.atan(sched.sigmas[0] / sched.config.sigma_data)
    out["decoder_1step"] = ns["_decoder_inference"](fake, (0, 2, -1), inp["dec_latents"].clone(), sched, ww, [t0], 128,
                                                    96).numpy()
    out["decoder_2step"] = ns["_decoder_inference"](fake, (0, 2, -1), inp["dec_latents"].clone(), sched, ww,
                                                    [t0, torch.arctan(torch.tensor(0.065) / 0.5)], 128, 96).numpy()
    # the product geometry (tile 512 / stride 384, world_pipeline.py:313-314), stored 4x sub-sampled to stay small
    ww512 = ns["linear_weight_window"](512, "cpu", torch.float32)
    full = ns["_decoder_inference"](fake, (0, -1, 3), inp["dec_latents_512"].clone(), sched, ww512, [t0], 512, 384)
    out["decoder_512_sub4"] = full[:, ::4, ::4].contiguous().numpy()
    del dec

    # ---------------- latent stage: batch of two windows, phase 1 (samples=None) then phase 2 on phase-1 output
    base = build(BASE_CFG)
    fake = SimpleNamespace(device=torch.device("cpu"), _dtype=None, seed=SEED, base_model=base, log_mode="quiet",
                           torch_compile=False)
    fake._process_latent_conditioning = functools.partial(ns["_process_latent_conditioning"], fake)
    ww64 = ns["linear_weight_window"](64, "cpu", torch.float32)
    ctxs = [(0, 1, 2), (0, -1, 0)]
    t_init = float(torch.atan(sched.sigmas[0] / sched.config.sigma_data))
    t_inter = float(torch.atan(torch.tensor(0.35) / 0.5))
    conds = [c.clone() for c in inp["lat_cond"]]
    p1 = ns["_latent_inference"](fake, ctxs, None, conds, t_init, sched, ww64, inp["lat_hist"], inp["lat_means"],
                                 inp["lat_stds"], seed_offset=offs[0])
    out["latent_phase1"] = torch.stack(p1).numpy()
    conds = [c.clone() for c in inp["lat_cond"]]
    p2 = ns["_latent_inference"](fake, ctxs, [p.clone() for p in p1], conds, t_inter, sched, ww64, inp["lat_hist"],
                                 inp["lat_means"], inp["lat_stds"], seed_offset=offs[1])
    out["latent_phase2"] = torch.stack(p2).numpy()
    out["latent_condvec"] = ns["_process_latent_conditioning"](
        fake, torch.cat([inp["lat_cond"][0][:-1] / inp["lat_cond"][0][-1:], torch.ones(1, 4, 4)])[None],
        inp["lat_hist"], inp["lat_means"], inp["lat_stds"], torch.tensor(0.0), seed_offset=65538).numpy()
    del base

    # ---------------- coarse stage: 20-step solve with five float conditions
    coarse = build(COARSE_CFG)
    fake = SimpleNamespace(device=torch.device("cpu"), _dtype=None, seed=SEED, coarse_model=coarse, log_mode="quiet",
                           kwargs={"coarse_means": inp["coarse_means"].tolist(),
                                   "coarse_stds": inp["coarse_stds"].tolist()},
                           _conditioning_model_input=lambda i1, i2, j1, j2: inp["coarse_map"].clone())
    t_cond = torch.atan(inp["cond_snr"])
    vals = torch.log(torch.tan(t_cond) / 8.0)
    cond_inputs = [v.detach().view(-1) for v in vals]
    out["coarse"] = ns["_coarse_inference"](fake, (0, 1, -2), EDMDPMSolverMultistepScheduler(
        sigma_min=0.002, sigma_max=80, sigma_data=0.5), ww64, t_cond, cond_inputs).numpy()
    np.savez_compressed(HERE / "stages_golden.npz", **out)
    print({k: (v.shape, float(np.abs(v).mean())) for k, v in out.items()})


if __name__ == "__main__":
    main()
