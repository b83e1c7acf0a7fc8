#!/usr/bin/env python
"""Cost of the batched coarse stage on one GPU, with the shipped coarse architecture (procedural weights) and a seeded
`conditioning_fn`.

    python tools/bench_coarse_batch.py [--iters 20] [--repeats 5] [--pools 1,2,4] [--out FILE]

It prints one JSON line, with the card's name, its enforced power limit and its SM clocks read in the same run, and
writes it to --out (default profiles/bench_coarse_batch.json):
  stage    the per-window cost of `coarse_stage_tiles` at n = 1, 2, 4, 8, 16 windows per call against
           `coarse_stage_tile` (one 20-step solve per call), host maps, host wall time to a device synchronise over
           `iters` calls, median of `repeats`.  Every batched window is compared bit for bit with its one-window solve.
  canvas   a cold `world.coarse[:, -50:50, -50:50]` (the generate CLI's default window) at every pool size with
           coarse_batch_size 1 and 16, the two alternating; the window cache is emptied before each timed read.
  land     a cold `world.land_tiles(300, 1024)` (the random sampler's default coarse window) with coarse_batch_size 1
           and 16, alternating.
Plans and graphs are built by warm-up calls first; the canvases compare bit for bit between the two batch sizes.
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

BATCHES = (1, 2, 4, 8, 16)


def gpu_query(index: int) -> dict:
    """Enforced power limit (W) and SM clocks (MHz: current, maximum), read-only nvidia-smi queries."""
    out = {"power_limit_w": None, "sm_clock_mhz": None, "sm_clock_max_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        lim, sm, smax = (float(v) for v in q.stdout.strip().split(","))
        out.update(power_limit_w=lim, sm_clock_mhz=sm, sm_clock_max_mhz=smax)
    except Exception:
        pass
    return out


def wall(fn, sync) -> float:
    t0 = time.perf_counter()
    fn()
    sync()
    return time.perf_counter() - t0


def run(args):
    import torch

    from oracle import unet as ounet
    from terrain_diffusion_b200.inference import WorldPipeline
    from terrain_diffusion_b200.inference.stages import coarse_stage_tile, coarse_stage_tiles
    from terrain_diffusion_b200.inference.tiling import linear_weight_window
    from terrain_diffusion_b200.models import EDMUnet2D
    from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
    from tests.test_oracle_golden import BASE_CFG, COARSE_CFG
    if not torch.cuda.is_available():
        raise SystemExit("bench_coarse_batch.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    sync = torch.cuda.synchronize
    pools = [int(s) for s in args.pools.split(",")]

    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.to(dev)

    def cond_fn(i1, i2, j1, j2):
        gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0x7FFFFFFF)
        return torch.randn(5, i2 - i1, j2 - j1, generator=gg)

    coarse, base, dec = build(COARSE_CFG), build(BASE_CFG), build(ounet.DECODER_CFG)

    # ---------------- (a) the stage: per-window cost at each batch size
    sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
    t_cond = torch.atan(torch.tensor([0.3, 0.1, 1.0, 0.1, 1.0]))
    cond_inputs = [v.view(-1) for v in torch.log(torch.tan(t_cond) / 8.0)]
    means, stds = [0.1, -0.4, 12.0, 3.0, 700.0, 20.0], [1.3, 0.7, 9.0, 4.0, 600.0, 15.0]
    ww = linear_weight_window(64, dev)
    ctxs = [(0, i, j) for i in range(-2, 2) for j in range(-2, 2)]
    maps = [cond_fn(i * 48, i * 48 + 64, j * 48, j * 48 + 64) for _, i, j in ctxs]
    one = lambda k: coarse_stage_tile(coarse, sched, 42, ctxs[k], maps[k], t_cond, cond_inputs, ww, means, stds)
    many = lambda n: coarse_stage_tiles(coarse, sched, 42, ctxs[:n], maps[:n], t_cond, cond_inputs, ww, means, stds)
    ref = [one(k) for k in range(16)]
    identical = True
    for n in BATCHES:
        got = many(n)
        identical &= all(torch.equal(g.view(torch.int32), r.view(torch.int32)) for g, r in zip(got, ref))
    sync()
    stage = {}
    one_times, many_times = [], {n: [] for n in BATCHES}
    for _ in range(args.repeats):           # alternate the variants inside every repeat
        one_times.append(wall(lambda: [one(k % 16) for k in range(args.iters)], sync) / args.iters)
        for n in BATCHES:
            many_times[n].append(wall(lambda: [many(n) for _ in range(args.iters)], sync) / args.iters / n)
    stage["coarse_stage_tile_ms_per_window"] = statistics.median(one_times) * 1e3
    stage["coarse_stage_tiles_ms_per_window"] = {str(n): statistics.median(v) * 1e3 for n, v in many_times.items()}
    stage["all_ms_per_window"] = {"coarse_stage_tile": [t * 1e3 for t in one_times],
                                  **{str(n): [t * 1e3 for t in v] for n, v in many_times.items()}}
    stage["bit_identical"] = bool(identical)
    stage["calls_per_repeat"] = args.iters

    # ---------------- (b) a cold coarse canvas read and (c) a cold land search, batch 1 against 16
    def world(pool, batch):
        w = WorldPipeline.from_local_models(coarse, base, dec, seed=42, coarse_pooling=pool, cache_limit=None,
                                            conditioning_fn=cond_fn, coarse_batch_size=batch).to(dev).bind()
        w.coarse[:, 100_000:100_200, 100_000:100_200]              # warm-up: plans, graphs, weight window
        sync()
        return w

    def cold(w, read):
        """One cold read: (host wall seconds to a device synchronise, coarse windows computed, the result)."""
        w.empty_cache()
        before = w._coarse.windows_computed
        t0 = time.perf_counter()
        out = read(w)
        sync()
        return time.perf_counter() - t0, w._coarse.windows_computed - before, out

    canvas = []
    for pool in pools:
        ws = {b: world(pool, b) for b in (1, 16)}
        res = {b: ([], 0, None) for b in ws}
        for _ in range(args.repeats):
            for b, w in ws.items():
                t, c, out = cold(w, lambda w: w.coarse[:, -50:50, -50:50])
                res[b] = (res[b][0] + [t], c, out)
        same = bool(torch.equal(res[1][2], res[16][2]))
        for b in ws:
            s = statistics.median(res[b][0])
            canvas.append({"coarse_pooling": pool, "coarse_batch_size": b, "windows": res[b][1], "wall_s": s,
                           "ms_per_window": s * 1e3 / res[b][1], "bit_identical_to_batch_1": same})
    ws = {b: world(1, b) for b in (1, 16)}
    res = {b: ([], 0, None) for b in ws}
    for _ in range(args.repeats):
        for b, w in ws.items():
            t, c, out = cold(w, lambda w: w.land_tiles(300, 1024))
            res[b] = (res[b][0] + [t], c, out)
    land = [{"coarse_batch_size": b, "windows": res[b][1], "wall_s": statistics.median(res[b][0]),
             "tiles_found": len(res[b][2]), "same_as_batch_1": res[b][2] == res[1][2]} for b in ws]

    line = {"metric": "coarse_batch_size: batched coarse-stage solves, cold coarse canvas and land search",
            "stage": stage,
            "canvas": {"window": "world.coarse[:, -50:50, -50:50]", "repeats": args.repeats, "results": canvas},
            "land": {"call": "world.land_tiles(300, 1024)", "coarse_pooling": 1, "repeats": args.repeats,
                     "results": land},
            "gpu": {"name": torch.cuda.get_device_name(dev), **gpu_query(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0))}, "torch": torch.__version__}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=20, help="timed stage calls per repeat and variant")
    ap.add_argument("--repeats", type=int, default=5, help="repeats (median) of every timed measurement")
    ap.add_argument("--pools", default="1,2,4", help="coarse_pooling values of the canvas read (default 1,2,4)")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_coarse_batch.json"),
                    help="write the JSON line here as well (default profiles/bench_coarse_batch.json)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
