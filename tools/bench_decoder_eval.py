#!/usr/bin/env python
"""The decoder evaluations on one GPU: `decoder_eval_terrain` on the two workloads of the original project's drivers,
the shipped 64x3 decoder with procedural weights, two TrigFlow steps (intermediate_sigma 0.065):

  * evaluation/decoder_consistency.py's defaults: batches of ten 512^2 images, one 512 tile each;
  * evaluation/tiled_decoder_consistency.py: batches of ten 896^2 images, 2 x 2 tiles of 512 at stride 384, the
    centre 512^2 crop (tile_batch 1: each program runs ten 512^2 tiles, as in the first workload).

    python tools/bench_decoder_eval.py [--images 10] [--steps 10] [--warmup 3]

Prints one JSON line with the card's name and enforced power limit read in the same run.  Inputs (the dataset's images,
pre-padded low-frequency planes and conditioning, a CUDA generator) are on the device.  Per workload, `value` =
images/s of decoder_eval_terrain; `baseline` = images/s of the drivers' loop as users run it today with the package's
EDMUnet2D dropped in: the tile loop, the TrigFlow update, the blend and the de-normalisation as torch ops, then the
pre-padded laplacian_decode, the signed square and the crop through the single-plane chain of inference/postproc.py,
plane by plane.  `readout` times the read-out of both terrains alone: one padded_terrain call over the 2B planes
against that per-plane chain.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench import ClockSampler  # noqa: E402
from bench_eval_samplers import power_limit_w  # noqa: E402
from bench_eval_terrain import timed  # noqa: E402

RESIDUAL_MEAN, RESIDUAL_STD, SIGMA_DATA = 0.0, 1.1678, 0.5     # consistency_decoder_64-3.cfg [results_dataset]
INTERMEDIATE_SIGMA = 0.065
WORKLOADS = {   # name: (image size, tile, stride, crop, tile_batch)
    "decoder_consistency": (512, 512, 256, None, None),
    "tiled_decoder_consistency": (896, 512, 384, 512, 1),
}


def per_plane(residual, lowfreq_padded, crop):
    """The single-plane read-out: laplacian_decode(pre_padded=True) + sign(x) x^2, then the centre crop."""
    from terrain_diffusion_b200.inference import postproc as P
    out = []
    for r, lo in zip(residual, lowfreq_padded):
        H, W = r.shape
        up = P.resize_bilinear(lo, (H + 16, W + 16))[8:8 + H, 8:8 + W]
        t = P._combine(r * RESIDUAL_STD + RESIDUAL_MEAN, up, signed_square=True)
        if crop:
            t = t[(H - crop) // 2:(H + crop) // 2, (W - crop) // 2:(W + crop) // 2]
        out.append(t)
    return torch.stack(out)[:, None]


def run_workload(name, args, model, dev, gen):
    from terrain_diffusion_b200.inference import decoder_eval_terrain, linear_weight_window, padded_terrain
    from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
    S, T, stride, crop, tile_batch = WORKLOADS[name]
    B, h = args.images, S // 8
    g = torch.Generator().manual_seed(11)
    images = (torch.randn(B, 1, S, S, generator=g) * SIGMA_DATA).to(dev)
    lowfreq_padded = (torch.randn(B, 1, h + 2, h + 2, generator=g) * 8 + 20).to(dev)
    cond_img = F.interpolate(torch.randn(B, 4, h, h, generator=g), size=(S, S), mode="nearest").to(dev)
    sch = EDMDPMSolverMultistepScheduler()

    def ours():
        return decoder_eval_terrain(model, sch, images, lowfreq_padded, cond_img, gen, residual_mean=RESIDUAL_MEAN,
                                    residual_std=RESIDUAL_STD, sigma_data=SIGMA_DATA, tile_size=T, tile_stride=stride,
                                    intermediate_sigma=INTERMEDIATE_SIGMA, crop_size=crop, tile_batch=tile_batch)

    # the drivers' loop (decoder_consistency.py:108-190) with the package's EDMUnet2D
    init_t = torch.tensor(np.arctan((sch.sigmas[0] / SIGMA_DATA).numpy()), device=dev)
    t_values = [init_t, torch.tensor(np.arctan(INTERMEDIATE_SIGMA / SIGMA_DATA), device=dev)]
    weights = linear_weight_window(T, dev)[None, None]

    def baseline():
        output, output_weights = torch.zeros(images.shape, device=dev), torch.zeros(images.shape, device=dev)
        n = (S - T) // stride + 1
        for i in range(n):
            for j in range(n):
                i0, j0 = i * stride, j * stride
                samples = torch.zeros((B, 1, T, T), device=dev)
                tile_cond = cond_img[..., i0:i0 + T, j0:j0 + T]
                for t_scalar in t_values:
                    t = t_scalar.view(1, 1, 1, 1).expand(B, 1, 1, 1).to(dtype=images.dtype)
                    z = torch.randn(samples.shape, generator=gen, device=dev) * SIGMA_DATA
                    x_t = torch.cos(t) * samples + torch.sin(t) * z
                    pred = -model(torch.cat([x_t / SIGMA_DATA, tile_cond], dim=1), t.flatten(), [])
                    samples = torch.cos(t) * x_t - torch.sin(t) * SIGMA_DATA * pred
                output[..., i0:i0 + T, j0:j0 + T] += samples * weights
                output_weights[..., i0:i0 + T, j0:j0 + T] += weights
        output = output / output_weights / SIGMA_DATA
        lp = lowfreq_padded[:, 0]
        return per_plane(output[:, 0], lp, crop), per_plane((images / SIGMA_DATA)[:, 0], lp, crop)

    with ClockSampler(dev.index) as clk:
        s_ours = timed(ours, args.steps, args.warmup, dev)
        s_base = timed(baseline, args.steps, args.warmup, dev)
        s_ours2 = timed(ours, args.steps, 1, dev)            # the spread: ours again, after the baseline
    residual = torch.cat([torch.randn(B, S, S, generator=g).to(dev), (images / SIGMA_DATA)[:, 0]])
    lp2 = torch.cat([lowfreq_padded[:, 0]] * 2)
    r_ours = timed(lambda: padded_terrain(residual, lp2, RESIDUAL_MEAN, RESIDUAL_STD, True, crop), 50, 5, dev)
    r_base = timed(lambda: per_plane(residual, lp2, crop), 50, 5, dev)
    same = torch.equal(padded_terrain(residual, lp2, RESIDUAL_MEAN, RESIDUAL_STD, True, crop)[:, None],
                       per_plane(residual, lp2, crop))
    s = min(s_ours, s_ours2)
    return {"value": B / s, "unit": "images/s", "ms_per_call": s * 1e3,
            "ms_per_call_repeat": [s_ours * 1e3, s_ours2 * 1e3],
            "config": {"images": B, "image": S, "tile": T, "stride": stride, "crop": crop, "tile_batch": tile_batch,
                       "intermediate_sigma": INTERMEDIATE_SIGMA},
            "clocks": clk.summary(),
            "baseline": {"value": B / s_base, "unit": "images/s", "ms_per_call": s_base * 1e3,
                         "api": "the drivers' tile loop with EDMUnet2D and torch ops + the per-plane read-out"},
            "speedup": s_base / s,
            "readout": {"planes": 2 * B, "batched_ms": r_ours * 1e3, "per_plane_ms": r_base * 1e3,
                        "speedup": r_base / r_ours, "bit_identical": same,
                        "api": "tdx_eval_padded_terrain vs postproc.resize_bilinear / _combine per plane"}}


def run(args):
    from oracle import unet as ounet
    from terrain_diffusion_b200.models import EDMUnet2D
    dev = torch.device("cuda", torch.cuda.current_device())
    model = EDMUnet2D(**ounet.DECODER_CFG).eval()
    model.load_state_dict(ounet.procedural_state_dict(ounet.DECODER_CFG, seed=0))
    model = model.to(dev)
    gen = torch.Generator(device=dev).manual_seed(548)
    with torch.no_grad():
        res = {name: run_workload(name, args, model, dev, gen) for name in WORKLOADS}
    first = res["decoder_consistency"]
    line = {"metric": "decoder evaluation images/sec (generated + real terrain per image), 64x3 decoder, two steps",
            "value": first["value"], "unit": "images/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
            "higher_is_better": True, "dtype": "bf16", "data": "synthetic",
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "workloads": res}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=10, help="images per batch (the drivers' --batch-size)")
    ap.add_argument("--steps", type=int, default=10, help="timed calls")
    ap.add_argument("--warmup", type=int, default=3, help="untimed calls first")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
