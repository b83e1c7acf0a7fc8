#!/usr/bin/env python
"""Consistency-base evaluation sampling on one GPU: the shape of the original project's evaluation/base_consistency.py
(253 M 192x3 base consistency model, procedural weights, batches of 40 images of one 64^2 tile, two TrigFlow phases:
t_0 = atan(sigma_0 / sigma_d) and intermediate_t 0.61).

    python tools/bench_eval_samplers.py [--images 40] [--steps 80] [--warmup 40]

Prints one JSON line in bench.py's format (it reuses bench.py's clock sampler and model config), with the card's name
and enforced power limit read in the same run.  One step = one phase of one image (one base-model forward on a 64^2
tile, 193.65 GFLOP).  `value` = steps/s of the two fused consistency programs and the re-noising launch between them,
replayed with the batch resident; `e2e` = the same through `sample_base_consistency` with the evaluation's arguments
(condition image, statistics and noise level on the device, a CUDA generator).  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from bench import BASE_CFG, GFLOP_PER_LATENT_PHASE, ClockSampler  # noqa: E402

EVAL_IMAGES, EVAL_TILE, EVAL_INTERMEDIATE_T = 40, 64, 0.61     # evaluation/base_consistency.py:175-187
GFLOP_PER_STEP = GFLOP_PER_LATENT_PHASE


def power_limit_w(index: int):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        return None


def run(args):
    from terrain_diffusion_b200.inference import sample_base_consistency
    from terrain_diffusion_b200.inference.samplers import _phase_times, get_consistency_solve
    from terrain_diffusion_b200.inference.stages import trig_mix
    from terrain_diffusion_b200.models import EDMUnet2D
    from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
    from oracle import unet as ounet
    dev = torch.device("cuda", torch.cuda.current_device())
    model = EDMUnet2D(**BASE_CFG).eval()
    model.load_state_dict(ounet.procedural_state_dict(BASE_CFG, seed=0))
    model = model.to(dev)
    B, T, sd = args.images, EVAL_TILE, 0.5
    sch = EDMDPMSolverMultistepScheduler()
    t0, t1 = _phase_times(sch, EVAL_INTERMEDIATE_T, torch.float32)
    g = torch.Generator().manual_seed(3)
    z0 = torch.randn(B, 5, T, T, generator=g).to(dev)
    z1 = torch.randn(B, 5, T, T, generator=g).to(dev)
    cvec = torch.randn(B, 58, generator=g).to(dev)
    first = get_consistency_solve(model, B, T, T, t0, sd, from_unit_noise=True)
    second = get_consistency_solve(model, B, T, T, t1, sd)
    for s in (first, second):
        s.prog.instantiate()

    def sample():
        s = first.run(z0, None, conditional_inputs=[cvec])
        return second.run(trig_mix(s, z1, math.cos(t1), math.sin(t1) * sd), None, conditional_inputs=[cvec])

    n_iter = max(1, -(-args.steps // 2))
    n_warm = max(1, -(-args.warmup // 2))
    for _ in range(n_warm):
        sample()
    torch.cuda.synchronize()
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device=dev)
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    with ClockSampler(dev.index) as clk:
        e0.record()
        for _ in range(n_iter):
            sample()
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    steps = n_iter * 2
    value = B * steps / (ms / 1e3)

    cond_img = torch.randn(B, 7, 4, 4, generator=g).to(dev)
    hist = torch.randn(B, 5, generator=g).to(dev)
    gen = torch.Generator(device=dev).manual_seed(5)

    def e2e():
        return sample_base_consistency(model, sch, (B, 5, T, T), cond_img, cond_means=torch.zeros(7, device=dev),
                                       cond_stds=torch.ones(7, device=dev), noise_level=torch.zeros(B, 1, device=dev),
                                       histogram_raw=hist, intermediate_t=EVAL_INTERMEDIATE_T, generator=gen,
                                       tile_size=T)
    e2e()
    torch.cuda.synchronize()
    t_start = time.perf_counter()
    for _ in range(n_iter):
        e2e()
    torch.cuda.synchronize()
    e2e_value = B * steps / (time.perf_counter() - t_start)

    first.prog.profile()
    msl, kinds = first.prog.profile()
    ig_ms = sum(m for m, k in zip(msl, kinds) if k == 1)
    n_ig = sum(1 for k in kinds if k == 1)
    share = ig_ms / sum(msl)
    step_ms = ms / steps
    achieved = GFLOP_PER_STEP * 1e9 * B / (step_ms * share / 1e3) / 1e12
    peak = 989.0   # H100 SXM data sheet, dense bf16 (a rated figure, not a measured one)
    roof = {"bound": "tensor", "kernel": "tdx::igemm_kernel (wgmma implicit-GEMM conv)", "achieved": achieved,
            "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak, "traffic": None, "launches": n_ig,
            "kernel_share_of_step": share, "avg_launch_us": step_ms * share / n_ig * 1e3,
            "method": "as bench.py's latent arm: per-launch CUDA events give the share, x graph-replayed step time"}
    line = {"metric": "consistency-base evaluation image-phases/sec, 64^2 latent tiles, base 253M U-Net",
            "value": value, "unit": "image-phases/s", "n_gpus": 1, "steps": steps, "warmup": n_warm * 2,
            "ms_per_step": step_ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16", "data": "synthetic",
            "config": {"workload": f"evaluation/base_consistency.py: {B} images x one 64x64 tile x 2 TrigFlow phases "
                                   f"(t_0, intermediate_t {EVAL_INTERMEDIATE_T})",
                       "images": B, "tile": T, "phases": 2, "intermediate_t": EVAL_INTERMEDIATE_T,
                       "gflop_per_step": GFLOP_PER_STEP},
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "clocks": clk.summary(),
            "e2e": {"value": e2e_value, "unit": "image-phases/s",
                    "api": "terrain_diffusion_b200.inference.sample_base_consistency"},
            "gpu_launches": (first.launches_per_solve + second.launches_per_solve + 1) * n_iter, "roofline": roof,
            "tflops": value * GFLOP_PER_STEP / 1e3}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=EVAL_IMAGES, help="images (one 64^2 tile each) sampled together")
    ap.add_argument("--steps", type=int, default=80, help="timed phases (rounded up to whole two-phase samples)")
    ap.add_argument("--warmup", type=int, default=40, help="warm-up phases (rounded up to whole samples)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
