#!/usr/bin/env python
"""River routing (`plot_flow_indicator` = D8 receivers + upstream counts + log1p) on one GPU at the sizes its callers
render: the explorer's 1024^2 detail view, 512^2 evaluation tiles and a 4096^2 (2^24 px, the largest allowed) window.

    python tools/bench_hydrology.py [--sizes 1024,512,4096] [--serpentine 512] [--iters 50] [--warmup 5]
                                    [--cpu-iters 2] [--out FILE]

For each size it prints, in one JSON line with the card's name and enforced power limit read in the same run:
  device_ms   per call with a CUDA tensor in and out: CUDA events around `iters` warm back-to-back calls (each call
              includes its 4-byte +-inf flag read-back);
  numpy_ms    per call with a numpy array in and out (host->device copy, the call, device->host copy), host clock;
  oracle_ms   per call of oracle/hydrology.py (vectorised numpy on the host; the CPU oracle the tests check against,
              not the reference, whose accumulation is a Python loop over every land pixel), host clock.
The terrain is a seeded smooth field with 1/8 of it NaN ocean.  `--serpentine n` adds the adversarial n x n ramp of
tests/_hydrology_inputs.py, whose single flow path of n^2/2 cells is the accumulation's worst case (its latency grows
with the longest path); it is timed over a few calls.  Writes nothing unless --out is given.
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


def measure(name, host, iters, warmup, cpu_iters, dev):
    import torch

    from oracle import hydrology as O
    from terrain_diffusion_b200.inference import plot_flow_indicator
    z = torch.from_numpy(host).to(dev)
    for _ in range(warmup):
        plot_flow_indicator(z)
        plot_flow_indicator(host)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = plot_flow_indicator(z)
    e1.record()
    torch.cuda.synchronize()
    device_ms = e0.elapsed_time(e1) / iters
    t0 = time.perf_counter()
    for _ in range(iters):
        out_np = plot_flow_indicator(host)
    numpy_ms = (time.perf_counter() - t0) * 1e3 / iters
    t0 = time.perf_counter()
    for _ in range(cpu_iters):
        ref = O.flow_indicator(host)
    oracle_ms = (time.perf_counter() - t0) * 1e3 / cpu_iters
    assert torch.equal(out.cpu(), torch.from_numpy(out_np))
    ulps = int(np.abs(out_np.view(np.int32).astype(np.int64) - ref.view(np.int32)).max())
    return {"case": name, "size": host.shape[0], "device_ms": device_ms, "numpy_ms": numpy_ms,
            "oracle_ms": oracle_ms, "max_ulps_vs_oracle": ulps, "max_count": float(np.expm1(ref.max())),
            "iters": iters, "mpix_per_s_device": host.size / device_ms / 1e3}


def run(args):
    import torch

    from tests._hydrology_inputs import serpentine, smooth_field
    if not torch.cuda.is_available():
        raise SystemExit("bench_hydrology.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    results = [measure("terrain", smooth_field(n, seed=n), args.iters, args.warmup, args.cpu_iters, dev)
               for n in [int(s) for s in args.sizes.split(",")]]
    if args.serpentine:
        z, path = serpentine(args.serpentine)
        r = measure("serpentine", z, 3, 1, 1, dev)
        r["longest_path_cells"] = len(path)
        results.append(r)
    line = {"metric": "river routing (plot_flow_indicator) per call", "unit": "ms", "warmup": args.warmup,
            "results": results,
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0)), "oracle_threads": "numpy, single-threaded"},
            "launches_per_call": 3, "memsets_per_call": 2}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="1024,512,4096", help="comma-separated square sizes (default: 1024,512,4096)")
    ap.add_argument("--serpentine", type=int, default=512,
                    help="size of the adversarial one-path ramp, even (default: 512; 0: skip)")
    ap.add_argument("--iters", type=int, default=50, help="timed calls per size on the GPU")
    ap.add_argument("--warmup", type=int, default=5, help="warm-up calls per size and input kind")
    ap.add_argument("--cpu-iters", type=int, default=2, help="timed calls of the CPU oracle per size")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
