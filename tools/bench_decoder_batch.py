#!/usr/bin/env python
"""Cost and device memory of the batched decoder stage on one GPU, with the shipped 64x3 consistency decoder (procedural
weights), the shipped coarse and base architectures and a seeded `conditioning_fn`.

    python tools/bench_decoder_batch.py [--iters 10] [--repeats 5] [--memory 1,2,4,8,16] [--worlds 1,2,4] [--out FILE]

It prints one JSON line, with the card's name, its enforced power limit and its SM clocks read in the same run, and
writes it to --out (default profiles/bench_decoder_batch.json):
  memory   per program size m of --memory, the device memory of the batch-invariant 512^2 decoder program (at m = 1
           the one-window program it shares with decoder_stage_tile): the bytes the torch allocator holds for it
           (activation arena, sample / condition buffers) and the drop in free device memory while it is built and
           first run (that also counts the CUDA graph and the library's workspaces; other processes on the card can
           move it).  Also the program's own run time per window (graph replay to a synchronise, median of
           `repeats` over `iters` runs), for sizes beyond DECODER_BATCH_SIZES too.
  split    the implicit-GEMM launches of the one-window 512^2 program that are split-K: at batch n a split-K launch
           runs as consecutive launches over window ranges, so these are where batch invariance costs throughput.
  stage    the per-window cost of `decoder_stage_tiles` at n = DECODER_BATCH_SIZES windows per call against
           `decoder_stage_tile`, 512^2 windows at stride 384, one consistency step: host wall time to a device
           synchronise over `iters` calls, median of `repeats`, the variants alternated.  Every batched window is
           compared bit for bit with its one-window solve.
  world    a cold `world.residual[:, 0:2048, 0:2048]` (the generate CLI's slice) and a cold 1024^2 `get()` with
           decoder_batch_size set to each of --worlds, coarse_batch_size 16 in every arm so only the decoder changes;
           alternated, every cache emptied before each timed read, results compared bit for bit.
Plans and graphs are built by warm-up calls first.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

TILE, STRIDE = 512, 384


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
    from terrain_diffusion_b200 import _lib as L
    from terrain_diffusion_b200.inference import WorldPipeline
    from terrain_diffusion_b200.inference.samplers import _solve_cache, get_consistency_solve
    from terrain_diffusion_b200.inference.stages import DECODER_BATCH_SIZES, decoder_stage_tile, decoder_stage_tiles
    from terrain_diffusion_b200.inference.tiling import linear_weight_window
    from terrain_diffusion_b200.models import EDMUnet2D
    from tests._capture import RecordingEmitter, RecordingProgram, folded, layer_of
    from tests.test_oracle_golden import BASE_CFG, COARSE_CFG
    if not torch.cuda.is_available():
        raise SystemExit("bench_decoder_batch.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    sync = torch.cuda.synchronize
    batches = list(DECODER_BATCH_SIZES)
    sizes = [int(s) for s in args.memory.split(",")]
    worlds = [int(s) for s in args.worlds.split(",")] if args.worlds else [1, *DECODER_BATCH_SIZES[-2:]]

    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.to(dev)

    def cond_fn(i1, i2, j1, j2):
        gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0x7FFFFFFF)
        return torch.randn(5, i2 - i1, j2 - j1, generator=gg)

    coarse, base, dec = build(COARSE_CFG), build(BASE_CFG), build(ounet.DECODER_CFG)
    sd = 0.5
    t0 = math.atan(80.0 / sd)                 # WorldPipeline.t_init: the one decoder step at sigma_max

    # ---------------- (a) device memory of the batch-invariant program at each size
    memory = []
    for m in sizes:
        _solve_cache(dec).clear()
        sync()
        torch.cuda.empty_cache()
        a0, (f0, _) = torch.cuda.memory_allocated(dev), torch.cuda.mem_get_info(dev)
        try:
            solve = get_consistency_solve(dec, m, TILE, TILE, t0, sd, from_unit_noise=True, out_scale=1 / sd,
                                          batch_invariant=m > 1)
            x, c = torch.randn_like(solve.sample), torch.randn_like(solve.cond)
            solve.run(x, c)
            sync()
        except (torch.cuda.OutOfMemoryError, L.TdxError) as e:
            memory.append({"m": m, "error": str(e).splitlines()[0]})
            _solve_cache(dec).clear()
            torch.cuda.empty_cache()
            continue
        a1, (f1, _) = torch.cuda.memory_allocated(dev), torch.cuda.mem_get_info(dev)
        times = [wall(lambda: [solve.run(x, c) for _ in range(args.iters)], sync) / args.iters / m
                 for _ in range(args.repeats)]
        memory.append({"m": m, "allocator_gb": (a1 - a0) / 1e9, "free_drop_gb": (f0 - f1) / 1e9,
                       "allocator_gb_per_window": (a1 - a0) / 1e9 / m,
                       "program_ms_per_window": statistics.median(times) * 1e3,
                       "all_program_ms_per_window": [t * 1e3 for t in times]})
        del solve, x, c
    _solve_cache(dec).clear()
    torch.cuda.empty_cache()

    # ---------------- (b) the split-K launches of the one-window plan
    fw = folded("decoder")
    prog = RecordingProgram()
    em = RecordingEmitter(fw, 1, TILE, TILE, prog)
    em.batch_invariant = True
    meta = torch.device("meta")
    em.emit_embed(prog, labels=torch.empty((1,), device=meta))
    em.emit(prog, [(torch.empty((1, fw.in_channels, TILE, TILE), device=meta), fw.in_channels, None)],
            model_out=torch.empty((1, fw.out_channels, TILE, TILE), device=meta))
    descs = prog.igemm()
    shapes = [L.igemm_launch_shape(d) for d in descs]
    split = [{"layer": layer_of(prog, d), "hw": int(d.height), "c_out": int(d.c_out), "n_item": s[0], "ksplit": s[1]}
             for d, s in zip(descs, shapes) if s[1] > 1]

    # ---------------- (c) the stage: per-window cost at each batch size
    ww = linear_weight_window(TILE, dev)
    g = torch.Generator().manual_seed(5)
    ctxs = [(0, i, j) for i in range(-2, 2) for j in range(-2, 2)]
    lats = [(torch.randn(6, TILE // 8, TILE // 8, generator=g) * 0.5).abs_().add_(0.1).to(dev) for _ in ctxs]
    one = lambda k: decoder_stage_tile(dec, 42, ctxs[k], lats[k], ww, [t0], TILE, STRIDE)
    many = lambda n: decoder_stage_tiles(dec, 42, ctxs[:n], lats[:n], ww, [t0], TILE, STRIDE)
    ref = [one(k) for k in range(len(ctxs))]
    identical = True
    for n in batches:
        got = many(n)
        identical &= all(torch.equal(x.view(torch.int32), r.view(torch.int32)) for x, r in zip(got, ref))
    sync()
    one_times, many_times = [], {n: [] for n in batches}
    for _ in range(args.repeats):           # alternate the variants inside every repeat
        one_times.append(wall(lambda: [one(k % len(ctxs)) for k in range(args.iters)], sync) / args.iters)
        for n in batches:
            many_times[n].append(wall(lambda: [many(n) for _ in range(args.iters)], sync) / args.iters / n)
    stage = {"decoder_stage_tile_ms_per_window": statistics.median(one_times) * 1e3,
             "decoder_stage_tiles_ms_per_window": {str(n): statistics.median(v) * 1e3 for n, v in many_times.items()},
             "all_ms_per_window": {"decoder_stage_tile": [t * 1e3 for t in one_times],
                                   **{str(n): [t * 1e3 for t in v] for n, v in many_times.items()}},
             "bit_identical": bool(identical), "calls_per_repeat": args.iters}
    del ref
    _solve_cache(dec).clear()
    torch.cuda.empty_cache()

    # ---------------- (d) cold reads of a world, decoder_batch_size 1 against the others
    def world(batch):
        w = WorldPipeline.from_local_models(coarse, base, dec, seed=42, cache_limit=None, conditioning_fn=cond_fn,
                                            coarse_batch_size=16, decoder_batch_size=batch,
                                            residual_mean=0.1, residual_std=1.2).to(dev).bind()
        w.residual[:, 100_000:102_048, 100_000:102_048]        # warm-up: plans and graphs of every padded size
        w.get(100_000, 100_000, 101_024, 101_024)
        sync()
        return w

    reads = {"residual_2048": lambda w: w.residual[:, 0:2048, 0:2048],
             "get_1024": lambda w: w.get(0, 0, 1024, 1024, with_climate=True)}
    ws = {b: world(b) for b in worlds}
    res = {(k, b): [] for k in reads for b in ws}
    outs, windows = {}, {}
    for _ in range(args.repeats):
        for k, read in reads.items():
            for b, w in ws.items():
                w.empty_cache()
                before = w._residual.windows_computed
                t = time.perf_counter()
                out = read(w)
                sync()
                res[(k, b)].append(time.perf_counter() - t)
                windows[(k, b)] = w._residual.windows_computed - before
                outs[(k, b)] = out
    world_rows = []
    for k in reads:
        for b in ws:
            a, r = outs[(k, b)], outs[(k, worlds[0])]
            same = (torch.equal(a.view(torch.int32), r.view(torch.int32)) if torch.is_tensor(a) else
                    all(torch.equal(a[q].view(torch.int32), r[q].view(torch.int32)) for q in ("elev", "climate")))
            world_rows.append({"read": k, "decoder_batch_size": b, "decoder_windows": windows[(k, b)],
                               "wall_s": statistics.median(res[(k, b)]), "all_wall_s": res[(k, b)],
                               f"bit_identical_to_batch_{worlds[0]}": bool(same)})

    line = {"metric": "decoder_batch_size: batched decoder-stage solves on 512^2 windows, program memory, cold reads",
            "memory": memory, "split_launches_one_window_512": split, "igemm_launches_per_forward": len(descs),
            "stage": stage,
            "world": {"reads": {"residual_2048": "world.residual[:, 0:2048, 0:2048]",
                                "get_1024": "world.get(0, 0, 1024, 1024, with_climate=True)"},
                      "coarse_batch_size": 16, "repeats": args.repeats, "results": world_rows},
            "gpu": {"name": torch.cuda.get_device_name(dev), **gpu_query(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0))}, "torch": torch.__version__}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=10, help="timed stage calls per repeat and variant")
    ap.add_argument("--repeats", type=int, default=5, help="repeats (median) of every timed measurement")
    ap.add_argument("--memory", default="1,2,4,8,16", help="program sizes whose memory and run time are measured")
    ap.add_argument("--worlds", default="", help="decoder_batch_size of the world arms, the first is the baseline "
                                               "(default: 1 and the two largest DECODER_BATCH_SIZES)")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_decoder_batch.json"),
                    help="write the JSON line here as well (default profiles/bench_decoder_batch.json)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
