"""Generate the golden fixtures in tests/golden/ from the UNMODIFIED reference (checkout at $TERRAIN_DIFFUSION_REF).

Run once in the build container (the reference cannot travel to the GPU box):
    python tests/golden/make_golden.py
Needs: $TERRAIN_DIFFUSION_REF, oracle/_stub (diffusers mixin stand-in, no arithmetic), numba.
Everything written here is small (inputs/outputs only; weights are re-created procedurally from names + seed by
oracle.unet.procedural_state_dict, identically here and in the tests).
"""
from __future__ import annotations

import ast
import os
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]

from terrain_diffusion.inference import portable_rng as ref_rng  # noqa: E402
from terrain_diffusion.models.edm_unet import EDMUnet2D  # noqa: E402
from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler  # noqa: E402
from terrain_diffusion.training.evaluation import _linear_weight_window, _tile_starts  # noqa: E402
from terrain_diffusion.training.evaluation.sample_diffusion_decoder import (  # noqa: E402
    sample_decoder_consistency_tiled, sample_decoder_diffusion_tiled)

from oracle import unet as O  # noqa: E402

torch.set_grad_enabled(False)

TINY_CFGS = {
    "tiny_dec": dict(image_size=32, in_channels=5, out_channels=1, model_channels=16, model_channel_mults=[1, 2],
                     layers_per_block=1, attn_resolutions=[], midblock_attention=False, concat_balance=0.5,
                     conditional_inputs=[], fourier_scale="pos"),
    "tiny_attn_cond": dict(image_size=16, in_channels=3, out_channels=3, model_channels=16,
                           model_channel_mults=[1, 2], layers_per_block=1, attn_resolutions=[8],
                           midblock_attention=True, concat_balance=0.3,
                           conditional_inputs=[["tensor", 7, 0.5], ["float", 8, 0.2], ["embedding", 5, 0.3]],
                           fourier_scale=1, block_kwargs={"channels_per_head": 8}),
}
BASE_CFG = dict(image_size=512, in_channels=5, out_channels=5, model_channels=192, model_channel_mults=[1, 2, 3, 4],
                layers_per_block=3, attn_resolutions=[8, 16], midblock_attention=True, concat_balance=0.5,
                conditional_inputs=[["tensor", 58, 1.0]], fourier_scale="pos", block_kwargs={"dropout": 0.1})
COARSE_CFG = dict(image_size=16, in_channels=11, out_channels=6, model_channels=128, model_channel_mults=[1],
                  layers_per_block=2, attn_resolutions=[], midblock_attention=False, concat_balance=0.5,
                  conditional_inputs=[["float", 64, 0.2]] * 5, fourier_scale="pos", block_kwargs={})


def build_ref(cfg, seed=0):
    m = EDMUnet2D(**cfg).eval()
    sd = O.procedural_state_dict(cfg, seed=seed)
    missing = set(m.state_dict()) ^ set(sd)
    assert not missing, missing
    m.load_state_dict(sd)
    return m, sd


def gen_inputs(cfg, n, hw, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, cfg["in_channels"], hw, hw, generator=g)
    t = torch.atan(torch.exp(torch.randn(n, generator=g) * 1.5) / 0.5)
    cond = []
    for kind, dim, _w in cfg.get("conditional_inputs") or []:
        if kind == "tensor":
            cond.append(torch.randn(n, dim, generator=g))
        elif kind == "float":
            cond.append(torch.randn(n, generator=g))
        else:
            cond.append(torch.randint(0, dim, (n,), generator=g))
    return x, t, cond


def golden_unets(out):
    for name, cfg in TINY_CFGS.items():
        m, _ = build_ref(cfg, seed=3)
        x, t, cond = gen_inputs(cfg, 2, cfg["image_size"], seed=11)
        out[f"{name}.y"] = m(x, t, cond).numpy()
    for name, cfg, hw in (("decoder", O.DECODER_CFG, 64), ("base", BASE_CFG, 64), ("coarse", COARSE_CFG, 64)):
        m, _ = build_ref(cfg, seed=0)
        x, t, cond = gen_inputs(cfg, 1, hw, seed=1)
        out[f"{name}.y"] = m(x, t, cond).numpy()
        print(name, "std", float(out[f"{name}.y"].std()))
        del m
    # one decoder forward at 128 with batch 2 (exercises every level at a non-trivial size)
    m, _ = build_ref(O.DECODER_CFG, seed=0)
    x, t, cond = gen_inputs(O.DECODER_CFG, 2, 128, seed=2)
    out["decoder128.y"] = m(x, t, cond).numpy()
    return m


def golden_scheduler(out):
    for n in (4, 12, 20):
        s = EDMDPMSolverMultistepScheduler()
        s.set_timesteps(n)
        out[f"sched{n}.sigmas"] = s.sigmas.numpy()
        out[f"sched{n}.timesteps"] = s.timesteps.numpy()
        g = torch.Generator().manual_seed(100 + n)
        x = torch.randn(1, 1, 8, 8, generator=g) * 80
        traj = []
        for t, sigma in zip(s.timesteps, s.sigmas):
            f = torch.randn(1, 1, 8, 8, generator=g)
            traj.append(torch.stack([s.precondition_inputs(x, sigma), f]))
            x = s.step(f, t, x).prev_sample
            traj.append(x.clone()[None].expand(2, -1, -1, -1, -1))
        out[f"sched{n}.traj"] = torch.stack(traj).numpy()
        out[f"sched{n}.cnoise"] = s.trigflow_precondition_noise(s.sigmas[:-1]).numpy()


def golden_tiling(out):
    cases = [(1664, 512, 384), (2048, 512, 384), (192, 64, 32), (896, 512, 384), (100, 64, 48), (64, 64, 64),
             (8192, 512, 384), (40, 64, 32), (65, 64, 64), (97, 32, 7)]
    out["tile_starts.cases"] = np.array(cases, dtype=np.int64)
    starts = [_tile_starts(*c) for c in cases]
    out["tile_starts.lens"] = np.array([len(s) for s in starts], dtype=np.int64)
    out["tile_starts.flat"] = np.array([v for s in starts for v in s], dtype=np.int64)
    for size in (4, 8, 64):
        out[f"window{size}"] = _linear_weight_window(size, torch.device("cpu"), torch.float32)[0, 0].numpy()
    w512 = _linear_weight_window(512, torch.device("cpu"), torch.float32)[0, 0]
    out["window512.probe"] = np.array([w512[0, 0], w512[0, 255], w512[255, 255], w512[511, 300], w512[17, 401]],
                                      dtype=np.float32)
    out["window512.sum64"] = np.array(w512.double().sum().item())


def golden_rng(out):
    for seed, n in ((42, 8), (1, 1000), (7046029251746621361, 4097), (0xFFFFFFFFFFFFFFFF, 257), (123456789, 65536)):
        out[f"normal.{seed}.{n}"] = ref_rng.standard_normal(seed, n, np.float32)
    out["normal64.1592590337.64"] = ref_rng.standard_normal(0x5EED0001, 64, np.float64)
    out["next_seed"] = np.array([ref_rng.next_seed(s) for s in (1, 42, 2 ** 63 + 5)], dtype=np.uint64)
    # _tile_seed / gaussian_noise_patch live in world_pipeline.py, which needs absent third-party packages to import;
    # execute just those two function definitions from the reference source in a scratch namespace.
    src = (REF / "terrain_diffusion/inference/world_pipeline.py").read_text()
    tree = ast.parse(src)
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("_tile_seed", "gaussian_noise_patch")]
    ns = {"np": np, "fill_standard_normal": ref_rng.fill_standard_normal}
    exec(compile(ast.Module(body=fns, type_ignores=[]), "world_pipeline_extract", "exec"), ns)
    seeds = [(1, 0, 0), (1, -1, 2), (123456789, 5, -7), (2 ** 64 - 1, -3, -3), (0, 2 ** 31, -2 ** 31)]
    out["tile_seed.args"] = np.array([[s % 2 ** 63, a, b] for s, a, b in seeds], dtype=np.int64)
    out["tile_seed.base_u64"] = np.array([s for s, _, _ in seeds], dtype=np.uint64)
    out["tile_seed.out"] = np.array([ns["_tile_seed"](*s) for s in seeds], dtype=np.uint64)
    patches = [(5, -10, -3, 24, 20, 2, 16, 16), (99, 0, 0, 16, 16, 1, 16, 16), (7, 30, -40, 9, 50, 3, 32, 8)]
    out["patch.args"] = np.array(patches, dtype=np.int64)
    for i, (seed, y0, x0, h, w, c, th, tw) in enumerate(patches):
        out[f"patch.{i}"] = ns["gaussian_noise_patch"](seed, y0, x0, h, w, c, th, tw)


def golden_samplers(out, decoder):
    g = torch.Generator().manual_seed(1)
    noise = torch.randn(1, 1, 64, 64, generator=g) * 80
    cond = torch.randn(1, 4, 64, 64, generator=g)
    sch = EDMDPMSolverMultistepScheduler()
    out["cfg1.y"] = sample_decoder_diffusion_tiled(decoder, sch, cond, noise, 64, 64, num_steps=4).numpy()
    # multi-tile consistency blend (stateless per tile): 96x96 canvas, tile 64, stride 32 -> 2x2 tiles
    g = torch.Generator().manual_seed(5)
    noise = torch.randn(1, 1, 96, 96, generator=g)
    cond = torch.randn(1, 4, 96, 96, generator=g)
    sch = EDMDPMSolverMultistepScheduler()
    out["consistency96.y"] = sample_decoder_consistency_tiled(decoder, sch, cond, noise, 64, 32,
                                                              intermediate_t=[0.6]).numpy()


def main():
    out: dict = {}
    decoder = golden_unets(out)
    golden_scheduler(out)
    golden_tiling(out)
    golden_rng(out)
    golden_samplers(out, decoder)
    np.savez_compressed(HERE / "reference_golden.npz", **out)
    sz = os.path.getsize(HERE / "reference_golden.npz")
    print(f"wrote {len(out)} arrays, {sz/1024:.0f} KiB")


if __name__ == "__main__":
    main()
