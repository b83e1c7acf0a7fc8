#!/usr/bin/env python
"""Shaded relief map (`get_relief_map`) on one GPU at the sizes its callers render: the explorer's 1024^2 detail view
(`/api/detail.png`) and the evaluations' 512^2 `--save-images` tiles.

    python tools/bench_relief.py [--sizes 1024,512] [--iters 200] [--warmup 20] [--cpu-iters 5] [--out FILE]

For each size it prints, in one JSON line with the card's name and enforced power limit read in the same run:
  device_ms   per call with a CUDA tensor in and out: CUDA events around `iters` warm back-to-back calls (each call
              includes its 4-byte NaN-count read-back);
  numpy_ms    per call with a numpy array in and out (host->device copy, the call, device->host copy), host clock;
  cpu_port_ms per call of oracle/relief.py (numpy + scipy on the host cores; a CPU port of the reference's function,
              not the reference itself, which needs matplotlib), host clock.
The elevation is a seeded smooth field with land and ocean.  Writes nothing unless --out is given.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402


def power_limit_w(index: int):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        return None


def elevation(n: int) -> np.ndarray:
    rng = np.random.RandomState(n)
    y, x = np.mgrid[0:n, 0:n].astype(np.float64) / n
    e = np.zeros((n, n))
    for _ in range(6):
        e += rng.uniform(300, 900) * np.sin(rng.uniform(2, 20) * y + rng.uniform(2, 20) * x + rng.uniform(0, 6.28))
    return (e + 200 + 30 * rng.randn(n, n)).astype(np.float32)


def run(args):
    import torch

    from oracle import relief as O
    from terrain_diffusion_b200.inference import get_relief_map
    if not torch.cuda.is_available():
        raise SystemExit("bench_relief.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    results = []
    for n in [int(s) for s in args.sizes.split(",")]:
        host = elevation(n)
        elev = torch.from_numpy(host).to(dev)
        for _ in range(args.warmup):
            get_relief_map(elev, None, None, None)
            get_relief_map(host, None, None, None)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            out = get_relief_map(elev, None, None, None)
        e1.record()
        torch.cuda.synchronize()
        device_ms = e0.elapsed_time(e1) / args.iters
        t0 = time.perf_counter()
        for _ in range(args.iters):
            out_np = get_relief_map(host, None, None, None)
        numpy_ms = (time.perf_counter() - t0) * 1e3 / args.iters
        t0 = time.perf_counter()
        for _ in range(args.cpu_iters):
            ref = O.relief_map(host)
        cpu_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters
        err = float(np.abs(out_np - ref).max())
        assert torch.equal(out.cpu(), torch.from_numpy(out_np))
        results.append({"size": n, "device_ms": device_ms, "numpy_ms": numpy_ms, "cpu_port_ms": cpu_ms,
                        "max_abs_diff_vs_cpu_port": err, "mpix_per_s_device": n * n / device_ms / 1e3})
    line = {"metric": "shaded relief map (get_relief_map) per call", "unit": "ms", "iters": args.iters,
            "warmup": args.warmup, "results": results,
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0)),
                     "cpu_port_threads": "numpy / scipy.ndimage, single-threaded for these operations"},
            "launches_per_call": 4}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="1024,512", help="comma-separated square sizes (default: 1024,512)")
    ap.add_argument("--iters", type=int, default=200, help="timed calls per size on the GPU")
    ap.add_argument("--warmup", type=int, default=20, help="warm-up calls per size and input kind")
    ap.add_argument("--cpu-iters", type=int, default=5, help="timed calls of the CPU port per size")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
