#!/usr/bin/env python
"""EDMAutoencoder on one GPU: the x8 autoencoder (configs/autoencoder/autoencoder_x8.cfg, 20.5 M parameters,
procedural weights) at the shapes the original project runs it at.

    python tools/bench_autoencoder.py [--steps 40] [--warmup 10]

  encode  `preencode` of the 8 flip / rotation variants of one 512^2 residual tile as one batch: the work
          data/preprocessing/build_encoded_dataset.py does per dataset tile
  decode  `decode` of 8 latents of 64^2 to 512^2

Prints one JSON line per workload in bench.py's format, with the card's name and enforced power limit read in the same
run.  `value` = tiles/s through the public call with the input and output on the device; `e2e` = the same with a host
tensor in and host tensors out.  GFLOP per tile is counted from the convolution shapes (conv_gflop below, the
algorithmic 2*Cin*Cout*k*k*H*W of every convolution; the im2col path's zero-padded K is not counted).  The implicit-GEMM
share of the forward comes from per-launch CUDA events of one eager replay, as in bench.py.  Writes nothing to disk.
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

TILES = 8          # the 8 flip / rotation variants of one tile (build_encoded_dataset.py)
TILE = 512


def conv_gflop(cfg: dict) -> dict:
    """GFLOP of one 512^2 tile through the encoder and through the decoder, from the planner's block lists."""
    from terrain_diffusion_b200.models.plan import autoencoder_decoder_plan, block_plan

    def conv(cin, cout, k, res):
        return 2.0 * cin * cout * k * k * res * res / 1e9

    enc_cfg = dict(cfg, encode_only=True)
    enc, _ = block_plan(enc_cfg)
    res, tot = TILE, 0.0
    for b in enc:
        if b["kind"] == "conv":
            tot += conv(b["cin"], b["cout"], 3, res)
            continue
        if b["resample"] == "down":
            res //= 2
        if b["cin"] != b["cout"]:
            tot += conv(b["cin"], b["cout"], 1, res)
        tot += 2 * conv(b["cout"], b["cout"], 3, res)
    tot += conv(enc[-1]["cout"], 2 * cfg["latent_channels"], 3, res)
    encode = tot
    first, dec = autoencoder_decoder_plan(cfg)
    tot = conv(first[0]["cin"], first[0]["cout"], 1, res)
    for b in dec:
        if b["resample"] == "up":
            res *= 2
        tot += conv(b["cin"], b["cout"], 3, res) + conv(b["cout"], b["cout"], 3, res)
        if b["cin"] != b["cout"]:
            tot += conv(b["cin"], b["cout"], 1, res)
    tot += conv(dec[-1]["cout"], cfg["out_channels"], 3, res)
    return {"encode": encode, "decode": tot}


def power_limit_w(index: int):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        return None


def flip_rot_variants(tile: torch.Tensor) -> torch.Tensor:
    """[8, 1, H, W]: the tile rotated by 0/90/180/270 degrees, without and with a horizontal flip."""
    out = []
    for flip in (False, True):
        t = torch.flip(tile, dims=[-1]) if flip else tile
        out += [torch.rot90(t, k, dims=(-2, -1)) for k in range(4)]
    return torch.stack(out)[:, None]


def run(args):
    from bench import ClockSampler
    from oracle import autoencoder as oae
    from terrain_diffusion_b200.models import EDMAutoencoder
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = oae.X8_CFG
    model = EDMAutoencoder(**cfg).eval()
    model.load_state_dict(oae.procedural_state_dict(cfg, seed=0))
    model = model.to(dev)
    gflop = conv_gflop(cfg)
    g = torch.Generator().manual_seed(3)
    x_host = flip_rot_variants(torch.randn(TILE, TILE, generator=g))
    z_host = torch.randn(TILES, cfg["latent_channels"], TILE // 8, TILE // 8, generator=g)
    x_dev, z_dev = x_host.to(dev), z_host.to(dev)
    lat = TILE // 8
    work = {
        "encode": (lambda: model.preencode(x_dev), lambda: [t.cpu() for t in model.preencode(x_host.to(dev))],
                   lambda: model.encoder._plans[("fwd", TILES, TILE, TILE, False)][0],
                   "build_encoded_dataset.py: preencode of the 8 flip/rotation variants of one 512x512 residual tile"),
        "decode": (lambda: model.decode(z_dev), lambda: model.decode(z_host.to(dev)).cpu(),
                   lambda: model._plans[("dec", TILES, lat, lat)][0],
                   f"decode of {TILES} latents of {lat}x{lat}x{cfg['latent_channels']} to {TILE}x{TILE}")}
    for name in args.workloads:
        fn, e2e_fn, prog_of, what = work[name]
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with ClockSampler(dev.index) as clk:
            e0.record()
            for _ in range(args.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        value = TILES / (ms / 1e3)
        e2e_fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            e2e_fn()
        torch.cuda.synchronize()
        e2e_value = TILES * args.steps / (time.perf_counter() - t0)
        prog = prog_of()
        prog.profile()                                     # warm the eager path
        msl, kinds = prog.profile()
        ig_ms = sum(m for m, k in zip(msl, kinds) if k == 1)
        n_ig = sum(1 for k in kinds if k == 1)
        share = ig_ms / sum(msl)
        achieved = gflop[name] * TILES / (ms * share / 1e3) / 1e3
        peak = 989.0   # H100 SXM data sheet, dense bf16 (a rated figure, not a measured one)
        roof = {"bound": "tensor", "kernel": "tdx::igemm_kernel (wgmma implicit-GEMM conv)", "achieved": achieved,
                "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak, "traffic": None, "launches": n_ig,
                "kernel_share_of_step": share, "avg_launch_us": ms * share / n_ig * 1e3,
                "method": "as bench.py: per-launch CUDA events of one eager replay give the share, x graph-replayed "
                          "call time"}
        line = {"metric": f"autoencoder {name} tiles/sec, {TILE}^2 tiles, x8 EDMAutoencoder",
                "value": value, "unit": "tiles/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "bf16", "data": "synthetic",
                "config": {"workload": what, "tiles_per_call": TILES, "tile": TILE, "gflop_per_tile": gflop[name]},
                "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
                "clocks": clk.summary(),
                "e2e": {"value": e2e_value, "unit": "tiles/s",
                        "api": f"terrain_diffusion_b200.models.EDMAutoencoder.{'preencode' if name == 'encode' else 'decode'}"
                               " (host tensor in, host tensors out)"},
                "gpu_launches": len(kinds), "roofline": roof,
                "tflops": value * gflop[name] / 1e3}
        print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=40, help="timed calls per workload")
    ap.add_argument("--warmup", type=int, default=10, help="warm-up calls per workload")
    ap.add_argument("--workloads", nargs="+", default=["encode", "decode"], choices=["encode", "decode"])
    run(ap.parse_args())


if __name__ == "__main__":
    main()
