#!/usr/bin/env python
"""The synthetic conditioning map and the Minecraft read-out's FastNoiseLite noise on the device (csrc/tdx_synth.cu)
against the host path.  pyfastnoiselite itself is not installed here, so the host side is the numpy restatement of the
same arithmetic (oracle/synthetic_map.py); pyfastnoiselite's own speed is not measured.

    python tools/bench_synthetic_map.py [--iters 50] [--cpu-iters 3] [--coarse-reps 5] [--out FILE]

Prints one JSON line with the card's name and enforced power limit read in the same run; medians of:
  window       one 5 x 64^2 conditioning window: `make_synthetic_map_factory(...)(i1, j1, i2, j2)` on the device (CUDA
               events; and host clock including the launch) against the oracle factory (host clock);
  minecraft    the five noise planes of a request at the sizes of tools/bench_minecraft_api.py (one tdx_fbm_perlin
               launch against the oracle), and the whole `/terrain` request at scale 2 with the noise included
               (`device_noise` against the oracle as `noise_fn`), on warm windows;
  coarse       a cold `world.coarse[:, -50:50, -50:50]` (nine 20-step coarse solves) of a WorldPipeline with
               `synthetic_map_stats=` against the same pipeline given the oracle factory as `conditioning_fn`,
               alternated in one run; every pair of results must be identical.
The statistics are the seeded fixture of tests/_synthetic_inputs.py.  Writes profiles/bench_synthetic_map.json unless
--out says otherwise.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tools")]


def device_ms(call, iters: int, warmup: int = 5) -> float:
    import torch
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    ev = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        ev.append((e0, e1))
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ev)


def host_ms(call, iters: int, sync: bool = False) -> float:
    import torch
    call()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        call()
        if sync:
            torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def build_models():
    import bench as B
    from oracle import unet as ounet
    from terrain_diffusion_b200.models import EDMUnet2D

    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.cuda()
    return build(B.COARSE_CFG), build(B.BASE_CFG), build(ounet.DECODER_CFG)


def run(args):
    import numpy as np
    import torch

    from bench_minecraft_api import power_limit_w, sm_clock_mhz
    from oracle import synthetic_map as O
    from terrain_diffusion_b200.inference import WorldPipeline
    from terrain_diffusion_b200.inference import minecraft as M
    from terrain_diffusion_b200.inference import postproc
    from terrain_diffusion_b200.inference import synthetic_map as S
    from tests._synthetic_inputs import FREQ_SYNTH, stats_mapping
    if not torch.cuda.is_available():
        raise SystemExit("bench_synthetic_map.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    stats = stats_mapping()
    out = {}

    # ---- one 5 x 64^2 window
    f = S.make_synthetic_map_factory(FREQ_SYNTH, 4242, stats=stats, device=dev)
    o = O.Factory(stats, FREQ_SYNTH, 4242)
    win = (-96, -32, -32, 32)
    out["window"] = {"cells": [5, 64, 64], "device_ms": device_ms(lambda: f(*win), args.iters),
                     "device_host_clock_ms": host_ms(lambda: f(*win), args.iters, sync=True),
                     "oracle_ms": host_ms(lambda: o(*win), args.cpu_iters),
                     "identical": bool(np.array_equal(f(*win).cpu().numpy(), o(*win)))}
    out["window"]["speedup"] = out["window"]["oracle_ms"] / out["window"]["device_host_clock_ms"]
    print(json.dumps(out["window"]), file=sys.stderr, flush=True)

    # ---- Minecraft noise planes and whole requests
    models = build_models()
    pipe = WorldPipeline.from_local_models(*models, seed=42, latents_batch_size=[1, 2, 4, 8, 16], cache_limit=None,
                                           synthetic_map_stats=stats).bind()
    nr = float(pipe.native_resolution)

    def oracle_noise(cfg, i0, j0, h, w):
        return O.fbm_plane(*cfg, i0, j0, h, w)

    mc = []
    for n in [int(s) for s in args.sizes.split(",")]:
        planes = torch.empty((5, n, n), dtype=torch.float32, device=dev)
        launch = lambda: S.fbm_planes(M.NOISE_CONFIGS, 3, 5, n, n, planes)   # noqa: E731
        host = lambda: np.stack([oracle_noise(c, 3, 5, n, n) for c in M.NOISE_CONFIGS])   # noqa: E731
        r = {"size": n, "noise_device_ms": device_ms(launch, args.iters), "noise_oracle_ms": host_ms(host, args.cpu_iters)}
        launch()
        r["noise_identical"] = bool(np.array_equal(planes.cpu().numpy(), host()))
        req = lambda fn: postproc.to_host(M.request(pipe._get_device, nr, 3, 5, 3 + n, 5 + n, 2, 1.0, fn,   # noqa: E731
                                                    payload=True)[0]).numpy().tobytes()
        body = req(M.device_noise)                                            # computes and caches the windows
        r["request_device_noise_ms"] = host_ms(lambda: req(M.device_noise), args.iters)
        r["request_oracle_noise_ms"] = host_ms(lambda: req(oracle_noise), args.cpu_iters)
        r["request_identical"] = body == req(oracle_noise)
        r["request_speedup"] = r["request_oracle_noise_ms"] / r["request_device_noise_ms"]
        mc.append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)
    out["minecraft"] = {"scale": 2, "noise": 1.0, "results": mc}

    # ---- cold coarse windows, device synthesis against the oracle as conditioning_fn, alternated
    host_pipe = None

    def cond_fn(i1, i2, j1, j2):
        return torch.from_numpy(O.Factory(stats, FREQ_SYNTH, host_pipe.seed)(j1, i1, j2, i2))

    host_pipe = WorldPipeline.from_local_models(*models, seed=42, cache_limit=None, conditioning_fn=cond_fn).bind()
    times = {"device": [], "host": []}
    identical = True
    for rep in range(args.coarse_reps + 1):
        got = {}
        for name, p in (("device", pipe), ("host", host_pipe)):
            p.empty_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got[name] = p.coarse[:, -50:50, -50:50]
            torch.cuda.synchronize()
            if rep:                                                            # rep 0 builds the solve programs
                times[name].append((time.perf_counter() - t0) * 1e3)
        identical = identical and torch.equal(got["device"], got["host"])
    out["coarse"] = {"window": [-50, 50, -50, 50], "solves": 9, "reps": args.coarse_reps,
                     "device_synthesis_ms": statistics.median(times["device"]),
                     "host_conditioning_fn_ms": statistics.median(times["host"]), "identical": bool(identical)}
    print(json.dumps(out["coarse"]), file=sys.stderr, flush=True)

    line = {"metric": "synthetic conditioning map and FastNoiseLite noise, device against the numpy restatement",
            "unit": "ms", "statistic": "median", "iters": args.iters, "cpu_iters": args.cpu_iters, **out,
            "pyfastnoiselite": "not installed: its own speed is not measured; the host side is oracle/synthetic_map.py",
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                    "clock_mhz": sm_clock_mhz(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0)), "numpy": np.__version__, "torch": torch.__version__}}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="16,256,1024", help="square Minecraft request sizes (default: 16,256,1024)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--cpu-iters", type=int, default=3)
    ap.add_argument("--coarse-reps", type=int, default=5)
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_synthetic_map.json"))
    run(ap.parse_args())


if __name__ == "__main__":
    main()
