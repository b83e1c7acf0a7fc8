#!/usr/bin/env python
"""Cost of `coarse_pooling` on one GPU, with the shipped coarse architecture (procedural weights) and a seeded
`conditioning_fn`.

    python tools/bench_coarse_pooling.py [--iters 2000] [--pools 1,2,4] [--repeats 3] [--out FILE]

It prints one JSON line, with the card's name and enforced power limit read in the same run, and writes it to --out
(default profiles/bench_coarse_pooling.json):
  epilogue   the coarse tile's epilogue for one tile: `tdx_coarse_epilogue` (one launch) against the op sequence it
             replaced (divide, multiply, add, the channel-1 subtract and its copy, `tdx_pack_weighted`), CUDA events
             around `iters` back-to-back launches; the fused epilogue also at every pool size.  At n = 1 the two
             outputs are compared bit for bit.
  canvas     a cold `world.coarse[:, -50:50, -50:50]` (the generate CLI's default window) at every pool size: the
             coarse windows computed and the host wall time to a device synchronise.  Plans and graphs are built by a
             warm-up read far away first; the window cache is emptied before each timed read; median of `repeats`.
             The number of coarse windows grows about as n^2.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def power_limit_w(index: int):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        pass
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(q.stdout.strip())
    except Exception:
        return None


def event_ms(fn, iters: int) -> float:
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def run(args):
    import torch

    from oracle import unet as ounet
    from terrain_diffusion_b200.inference import WorldPipeline, coarse_epilogue
    from terrain_diffusion_b200.inference.stages import pack_weighted
    from terrain_diffusion_b200.inference.tiling import linear_weight_window
    from terrain_diffusion_b200.models import EDMUnet2D
    from tests.test_oracle_golden import BASE_CFG, COARSE_CFG
    if not torch.cuda.is_available():
        raise SystemExit("bench_coarse_pooling.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    pools = [int(s) for s in args.pools.split(",")]

    # ---------------- (a) the epilogue of one tile
    g = torch.Generator().manual_seed(0)
    sample = (torch.randn(1, 6, 64, 64, generator=g) * 3).to(dev)
    means, stds = torch.randn(6, generator=g).to(dev), (torch.rand(6, generator=g) + 0.5).to(dev)

    def old():
        out = sample / 0.5 * stds.view(1, -1, 1, 1) + means.view(1, -1, 1, 1)
        out[:, 1] = out[:, 0] - out[:, 1]
        return pack_weighted(out.contiguous(), linear_weight_window(64, dev))

    fused = {n: (lambda n=n: coarse_epilogue(sample, means, stds, linear_weight_window(64 // n, dev), n, "max", "min"))
             for n in sorted(set(pools) | {1, 2, 4, 8, 16})}
    identical = bool(torch.equal(old().view(torch.int32), fused[1]().view(torch.int32)))
    for _ in range(args.warmup):
        old()
        for f in fused.values():
            f()
    torch.cuda.synchronize()
    old_ms = min(event_ms(old, args.iters) for _ in range(3))
    fused_ms = {n: min(event_ms(f, args.iters) for _ in range(3)) for n, f in fused.items()}
    epilogue = {"old_op_sequence_us": old_ms * 1e3, "old_launches": 6, "fused_us": {str(n): v * 1e3
                                                                                  for n, v in fused_ms.items()},
                "fused_launches": 1, "n1_bit_identical": identical, "iters": args.iters}

    # ---------------- (b) a cold coarse canvas read at each pool size
    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.to(dev)

    def cond_fn(i1, i2, j1, j2):
        gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0x7FFFFFFF)
        return torch.randn(5, i2 - i1, j2 - j1, generator=gg)

    coarse, base, dec = build(COARSE_CFG), build(BASE_CFG), build(ounet.DECODER_CFG)
    canvas = []
    for n in pools:
        world = WorldPipeline.from_local_models(coarse, base, dec, seed=42, coarse_pooling=n,
                                                elev_coarse_pool_mode="max", p5_coarse_pool_mode="min",
                                                cache_limit=None, conditioning_fn=cond_fn).to(dev).bind()
        world.coarse[:, 100_000:100_001, 100_000:100_001]            # warm-up: plan, graph, weight window
        torch.cuda.synchronize()
        times, counts = [], []
        for _ in range(args.repeats):
            world.empty_cache()
            before = world._coarse.windows_computed
            t0 = time.perf_counter()
            out = world.coarse[:, -50:50, -50:50]                      # a host view: ends in a device-to-host copy
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            counts.append(world._coarse.windows_computed - before)
        assert out.shape == (7, 100, 100) and bool(torch.isfinite(out).all())
        s = statistics.median(times)
        canvas.append({"coarse_pooling": n, "windows": counts[0], "wall_s": s, "ms_per_window": s * 1e3 / counts[0],
                       "wall_s_all": times})
    line = {"metric": "coarse_pooling: coarse-tile epilogue and cold coarse canvas read",
            "epilogue": epilogue, "canvas": {"window": "world.coarse[:, -50:50, -50:50]", "repeats": args.repeats,
                                             "modes": ["max", "min"], "results": canvas},
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0))}, "torch": torch.__version__}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=2000, help="timed epilogue launches per measurement")
    ap.add_argument("--warmup", type=int, default=50, help="warm-up epilogue launches per variant")
    ap.add_argument("--pools", default="1,2,4", help="coarse_pooling values of the canvas read (default 1,2,4)")
    ap.add_argument("--repeats", type=int, default=3, help="timed cold canvas reads per pool size")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_coarse_pooling.json"),
                    help="write the JSON line here as well (default profiles/bench_coarse_pooling.json)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
