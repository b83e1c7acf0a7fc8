#!/usr/bin/env python
"""Two-model guided base diffusion on one GPU: the shape of the original project's evaluation/base_diffusion.py (192x3
main U-Net + 128x3 guide, procedural weights, batches of 64^2 tiles, 32-step DPM-Solver++, guidance 2.15).

    python tools/bench_guided.py [--tiles 40] [--solve-steps 32] [--steps 64] [--warmup 32]

Prints one JSON line in bench.py's format (it reuses bench.py's clock sampler and model configs).  One step = the main
and guide forwards plus the guided update of one tile; `value` = tile-steps/s of the fused solve replayed with the
batch resident, `e2e` = the same through `sample_base_diffusion` with host inputs, `roofline` = the implicit-GEMM
kernel's share of the step (per-launch CUDA events) against the data-sheet dense bf16 rate, with the GFLOP per step
computed from the conv / attention shapes (unet_gflop).  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from bench import BASE_CFG, ClockSampler  # noqa: E402

GUIDE_CFG = dict(BASE_CFG, model_channels=128)
"""The 128x3 guide of evaluation/base_diffusion.py:105-122 (common/model_utils.py:10-11: diffusion_base_guide)."""
GUIDED_SCALE, GUIDED_STEPS, GUIDED_TILES = 2.15, 32, 40     # evaluation/base_diffusion.py:183-199


def unet_gflop(cfg: dict, hw: int) -> float:
    """Dense FLOPs (2 x MACs) of one U-Net forward on an hw x hw input, from the conv / attention shapes of the
    block plan: first conv, per block [1x1 skip conv] + two 3x3 convs [+ qkv / proj 1x1 convs + the two attention
    matmuls], last conv.  Embedding linears are negligible and not counted."""
    from terrain_diffusion_b200.models.plan import block_plan
    enc, dec = block_plan(cfg)

    def conv(ci, co, k, s):
        return 2.0 * ci * co * k * k * s * s

    def attn(c, s):
        return conv(c, 3 * c, 1, s) + conv(c, c, 1, s) + 2 * 2.0 * (s * s) ** 2 * c

    tot, s = 0.0, hw
    for b in enc:
        if b["kind"] == "conv":
            tot += conv(b["cin"], b["cout"], 3, s)
            continue
        if b["resample"] == "down":
            s //= 2
        tot += (conv(b["cin"], b["cout"], 1, s) if b["cin"] != b["cout"] else 0.0) + 2 * conv(b["cout"], b["cout"], 3, s)
        tot += attn(b["cout"], s) if b["attention"] else 0.0
    for b in dec:
        if b["resample"] == "up":
            s *= 2
        tot += conv(b["cin"], b["cout"], 3, s) + conv(b["cout"], b["cout"], 3, s)
        tot += (conv(b["cin"], b["cout"], 1, s) if b["cin"] != b["cout"] else 0.0)
        tot += attn(b["cout"], s) if b["attention"] else 0.0
    tot += conv(dec[-1]["cout"], cfg.get("out_channels") or cfg["in_channels"], 3, s)
    return tot / 1e9


def run(args):
    """Two-model guided base diffusion (evaluation/base_diffusion.py: 192x3 main + 128x3 guide, batches of 64^2
    tiles, guidance 2.15).  A step = the main and guide forwards plus the guided DPM-Solver++ update of one tile;
    `value` replays the fused solve (both models, every step, one graph) with the batch resident, `e2e` goes through
    `sample_base_diffusion` with host condition vectors and a host generator."""
    from terrain_diffusion_b200.inference import sample_base_diffusion
    from terrain_diffusion_b200.inference.samplers import get_diffusion_solve
    from terrain_diffusion_b200.models import EDMUnet2D
    from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
    from oracle import unet as ounet
    dev = torch.device("cuda", torch.cuda.current_device())
    models = []
    for cfg, seed in ((BASE_CFG, 0), (GUIDE_CFG, 1)):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=seed))
        models.append(m.to(dev))
    model, guide = models
    B, K, T = args.tiles, args.solve_steps, 64
    sch = EDMDPMSolverMultistepScheduler()
    g = torch.Generator().manual_seed(3)
    noise = (torch.randn(B, 5, T, T, generator=g) * 80.0).to(dev)
    cvec = torch.randn(B, 58, generator=g)
    cvec_d = cvec.to(dev)
    solve = get_diffusion_solve(model, sch, B, T, T, K, guide=guide, guidance_scale=GUIDED_SCALE)
    solve.prog.instantiate()
    n_solves = max(1, -(-args.steps // K))
    for _ in range(max(1, -(-args.warmup // K))):
        solve.run(noise, None, conditional_inputs=[cvec_d])
    torch.cuda.synchronize()
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device=dev)
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    with ClockSampler(dev.index) as clk:
        e0.record()
        for _ in range(n_solves):
            solve.run(noise, None, conditional_inputs=[cvec_d])
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    steps = n_solves * K
    value = B * steps / (ms / 1e3)
    e2e_value, e2e_err = None, None
    try:
        def e2e():
            y = sample_base_diffusion(model, sch, (B, 5, T, T), [cvec], cond_means=None, cond_stds=None,
                                      histogram_raw=None, steps=K, guide_model=guide, guidance_scale=GUIDED_SCALE,
                                      generator=torch.Generator().manual_seed(5))
            return y.cpu()
        e2e()
        n_e = 2
        t0 = time.perf_counter()
        for _ in range(n_e):
            e2e()
        e2e_value = B * K * n_e / (time.perf_counter() - t0)
    except Exception as exc:                                       # the kernel-only number stands on its own
        e2e_err = repr(exc)
    gflop_step = unet_gflop(BASE_CFG, T) + unet_gflop(GUIDE_CFG, T)
    solve.prog.profile()
    msl, kinds = solve.prog.profile()
    ig_ms = sum(m for m, k in zip(msl, kinds) if k == 1)
    n_ig = sum(1 for k in kinds if k == 1)
    share = ig_ms / sum(msl)
    step_ms = ms / steps
    achieved = gflop_step * 1e9 * B / (step_ms * share / 1e3) / 1e12
    peak = 989.0   # H100 SXM data sheet, dense bf16 (a rated figure, not a measured one)
    roof = {"bound": "tensor", "kernel": "tdx::igemm_kernel (wgmma implicit-GEMM conv)", "achieved": achieved,
            "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak, "traffic": None, "launches": n_ig,
            "kernel_share_of_step": share, "avg_launch_us": step_ms * share / (n_ig / K) * 1e3,
            "method": "as bench.py's latent arm: per-launch CUDA events give the share, x graph-replayed step time"}
    line = {"metric": "guided base-diffusion tile-steps/sec, 64^2 tiles, 192x3 main + 128x3 guide", "value": value,
            "unit": "tile-steps/s", "n_gpus": 1, "steps": steps, "warmup": max(1, -(-args.warmup // K)) * K,
            "ms_per_step": step_ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16", "data": "synthetic",
            "config": {"workload": f"evaluation/base_diffusion.py: {B} x 64x64 tiles, {K}-step DPM-Solver++ with "
                                   f"two-model guidance {GUIDED_SCALE} (main and guide forward per step, fused update)",
                       "tiles_per_gpu": B, "tile": T, "solve_steps": K, "guidance_scale": GUIDED_SCALE,
                       "gflop_per_tile_step": gflop_step},
            "clocks": clk.summary(),
            "e2e": {"value": e2e_value, "unit": "tile-steps/s", "error": e2e_err,
                    "api": "terrain_diffusion_b200.inference.sample_base_diffusion"},
            "gpu_launches": solve.launches_per_solve * n_solves, "roofline": roof,
            "tflops": value * gflop_step / 1e3}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=GUIDED_TILES, help="64^2 tiles solved together")
    ap.add_argument("--solve-steps", type=int, default=GUIDED_STEPS, help="DPM-Solver++ steps per solve")
    ap.add_argument("--steps", type=int, default=64, help="timed steps (rounded up to whole solves)")
    ap.add_argument("--warmup", type=int, default=32, help="warm-up steps (rounded up to whole solves)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
