#!/usr/bin/env python
"""The evaluation drivers' terrain decode on one GPU: `decode_latents_to_terrain` in the shape of the original
project's evaluation/base_consistency.py (decoder_batch_size 10: ten 64^2 base samples -> ten 512^2 terrains, the
shipped 64x3 decoder with procedural weights, two TrigFlow phases at atan(sigma_0 / sigma_d) and inter_t 0.13,
Laplacian denoising on).

    python tools/bench_eval_terrain.py [--images 10] [--steps 20] [--warmup 5]

Prints one JSON line with the card's name and enforced power limit read in the same run.  Inputs (samples, dataset
statistics, a CUDA generator) are on the device.  `value` = images/s of decode_latents_to_terrain; `baseline` = images/s
of the same decode composed from the package's public functions as they stood before it: sample_decoder_consistency_tiled
(one tile per image) and the single-plane laplacian_denoise / laplacian_decode per image.  `readout` times the read-out
alone: the batched tdx_eval_terrain against that per-plane chain.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_eval_samplers import power_limit_w  # noqa: E402

EVAL_IMAGES, EVAL_LATENT, EVAL_INTER_T = 10, 64, 0.13      # evaluation/base_consistency.py:79, 175-195


class Stats:
    def __init__(self, dev):
        self.latents_mean = torch.tensor([0.1, -0.2, 0.05, 0.3], device=dev).view(1, 4, 1, 1)
        self.latents_std = torch.tensor([1.2, 0.8, 1.5, 0.9], device=dev).view(1, 4, 1, 1)
        self.residual_mean, self.residual_std = 0.25, 1.75


def timed(fn, steps: int, warmup: int, dev) -> float:
    """Seconds per call: CUDA events around `steps` calls after `warmup` untimed ones."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize(dev)
    return e0.elapsed_time(e1) / 1e3 / steps


def run(args):
    from oracle import unet as ounet
    from terrain_diffusion_b200.inference import decode_latents_to_terrain, sample_decoder_consistency_tiled
    from terrain_diffusion_b200.inference import postproc as P
    from terrain_diffusion_b200.inference.evaluation import eval_terrain
    from terrain_diffusion_b200.models import EDMUnet2D
    from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
    dev = torch.device("cuda", torch.cuda.current_device())
    model = EDMUnet2D(**ounet.DECODER_CFG).eval()
    model.load_state_dict(ounet.procedural_state_dict(ounet.DECODER_CFG, seed=0))
    model = model.to(dev)
    B, h = args.images, EVAL_LATENT
    H = 8 * h
    g = torch.Generator().manual_seed(3)
    samples = torch.randn(B, 5, h, h, generator=g).to(dev)
    ds = Stats(dev)
    sch = EDMDPMSolverMultistepScheduler()
    gen = torch.Generator(device=dev).manual_seed(5)

    def ours():
        return decode_latents_to_terrain(samples, ds, model, sch, gen, [EVAL_INTER_T])

    def per_plane(residual, lowfreq):
        out = []
        for r, lo in zip(residual, lowfreq):
            r = r * ds.residual_std + ds.residual_mean
            lo = lo * P.LOWFREQ_STD + P.LOWFREQ_MEAN
            r, lo = P.laplacian_denoise(r, lo, 5)
            out.append(P.laplacian_decode(r, lo, extrapolate=True))
        return torch.stack(out)[:, None]

    def baseline():
        cond = F.interpolate(samples[:, :4] / ds.latents_std + ds.latents_mean, size=(H, H), mode="nearest")
        noise = torch.randn((B, 1, H, H), generator=gen, device=dev)
        residual = sample_decoder_consistency_tiled(model, sch, cond, noise, H, H, intermediate_t=[EVAL_INTER_T])
        return per_plane(residual[:, 0], samples[:, 4])

    with ClockSampler(dev.index) as clk:
        s_ours = timed(ours, args.steps, args.warmup, dev)
        s_base = timed(baseline, args.steps, args.warmup, dev)
        s_ours2 = timed(ours, args.steps, 1, dev)            # the spread: ours again, after the baseline
    residual = torch.randn(B, H, H, generator=g).to(dev)
    lowfreq = samples[:, 4].contiguous()
    r_ours = timed(lambda: eval_terrain(residual, lowfreq, ds.residual_mean, ds.residual_std), 50, 5, dev)
    r_base = timed(lambda: per_plane(residual, lowfreq), 50, 5, dev)
    same = torch.equal(eval_terrain(residual, lowfreq, ds.residual_mean, ds.residual_std)[:, None],
                       per_plane(residual, lowfreq))
    value = B / min(s_ours, s_ours2)
    line = {"metric": "evaluation terrain decode images/sec, 64^2 base samples -> 512^2 terrain, 64x3 decoder",
            "value": value, "unit": "images/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "ms_per_call": min(s_ours, s_ours2) * 1e3, "ms_per_call_repeat": [s_ours * 1e3, s_ours2 * 1e3],
            "higher_is_better": True, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": f"evaluation/base_consistency.py _decode_latents_to_terrain: {B} images of "
                                   f"{h}x{h} latents, inter_t [{EVAL_INTER_T}], Laplacian denoising on",
                       "images": B, "latent": h, "image": H, "inter_t": [EVAL_INTER_T]},
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "clocks": clk.summary(),
            "baseline": {"value": B / s_base, "unit": "images/s", "ms_per_call": s_base * 1e3,
                         "api": "sample_decoder_consistency_tiled + per-image laplacian_denoise / laplacian_decode"},
            "speedup": s_base / min(s_ours, s_ours2),
            "readout": {"batched_ms": r_ours * 1e3, "per_plane_ms": r_base * 1e3, "speedup": r_base / r_ours,
                        "bit_identical": same, "api": "tdx_eval_terrain vs postproc.laplacian_denoise / decode"}}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=EVAL_IMAGES, help="images decoded per call (decoder_batch_size)")
    ap.add_argument("--steps", type=int, default=20, help="timed calls")
    ap.add_argument("--warmup", type=int, default=5, help="untimed calls first")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
