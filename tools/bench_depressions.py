#!/usr/bin/env python
"""Depression fill (`fill_depressions_priority_flood`) and river-bed smoothing (`smooth_river_bumps`) on one GPU at
the sizes their callers render: 512^2 evaluation tiles, the explorer's 1024^2 detail view and a 4096^2 (2^24 px, the
largest allowed) window, plus the fill's worst case.

    python tools/bench_depressions.py [--sizes 512,1024,4096] [--serpentine 512] [--iters 20] [--warmup 3]
                                      [--cpu-iters 1] [--oracle-max 1024] [--out FILE]

For each size it prints, in one JSON line with the card's name and enforced power limit read in the same run:
  fill_device_ms    per call with a CUDA tensor in and out: CUDA events around `iters` warm back-to-back calls (each
                    call reads one flag word back per batch of relaxation passes);
  fill_numpy_ms     per call with a numpy array in and out (host->device copy, the call, device->host copy);
  passes            relaxation passes the call ran, the last one lowering nothing;
  oracle_ms         per call of oracle/depressions.py on the host (the Jacobi restatement for terrain, the ordered
                    heap one for the serpentine), and `equal_to_oracle`, the bit-for-bit comparison; both null above
                    --oracle-max, where the host oracle would take minutes;
  smooth_device_ms  smooth_river_bumps with the default three iterations, CUDA tensor in and out.
The terrain is a seeded smooth field with 1/8 of it NaN ocean.  `--serpentine n` adds the adversarial n x n flat of
tests/_depression_inputs.py: one outlet and one raised chain of about n^2/2 cells, the fill's longest dependency
chain.  Writes nothing unless --out is given.
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


def device_ms(fn, iters):
    import torch
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, out


def measure(name, host, iters, warmup, cpu_iters, oracle_max, dev, ordered=False):
    import torch

    from oracle import depressions as O
    from terrain_diffusion_b200.inference import fill_depressions_priority_flood, smooth_river_bumps
    from terrain_diffusion_b200.inference import hydrology as H
    z = torch.from_numpy(host).to(dev)
    for _ in range(warmup):
        fill_depressions_priority_flood(z)
        fill_depressions_priority_flood(host)
        smooth_river_bumps(z)
    fill_ms, out = device_ms(lambda: fill_depressions_priority_flood(z), iters)
    smooth_ms, _ = device_ms(lambda: smooth_river_bumps(z), iters)
    t0 = time.perf_counter()
    for _ in range(iters):
        out_np = fill_depressions_priority_flood(host)
    numpy_ms = (time.perf_counter() - t0) * 1e3 / iters
    assert np.array_equal(out.cpu().numpy().view(np.uint32), out_np.view(np.uint32))
    _, passes = H._fill(z.contiguous(), float(np.float32(1e-3)), 8, float("nan"))
    oracle_ms = equal = None
    if host.shape[0] <= oracle_max:
        t0 = time.perf_counter()
        for _ in range(cpu_iters):
            ref = O.fill_ordered(host) if ordered else O.fill(host)[0]
        oracle_ms = (time.perf_counter() - t0) * 1e3 / cpu_iters
        equal = bool(np.array_equal(ref.view(np.uint32), out_np.view(np.uint32)))
    return {"case": name, "size": host.shape[0], "fill_device_ms": fill_ms, "fill_numpy_ms": numpy_ms,
            "passes": passes, "oracle_ms": oracle_ms, "oracle": "ordered heap" if ordered else "jacobi",
            "equal_to_oracle": equal, "raised_px": int((out_np > host).sum()), "smooth_device_ms": smooth_ms,
            "iters": iters}


def run(args):
    import torch

    from tests._depression_inputs import fill_serpentine
    from tests._hydrology_inputs import smooth_field
    if not torch.cuda.is_available():
        raise SystemExit("bench_depressions.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    results = [measure("terrain", smooth_field(n, seed=n), args.iters, args.warmup, args.cpu_iters, args.oracle_max,
                       dev) for n in [int(s) for s in args.sizes.split(",")]]
    if args.serpentine:
        z, chain = fill_serpentine(args.serpentine)
        r = measure("serpentine", z, 3, 1, 1, args.oracle_max, dev, ordered=True)
        r["chain_cells"] = chain
        results.append(r)
    line = {"metric": "depression fill / river smoothing per call", "unit": "ms", "warmup": args.warmup,
            "results": results,
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0)), "oracle_threads": "numpy, single-threaded"}}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="512,1024,4096", help="comma-separated square sizes (default: 512,1024,4096)")
    ap.add_argument("--serpentine", type=int, default=512,
                    help="size of the adversarial one-chain flat, even (default: 512; 0: skip)")
    ap.add_argument("--iters", type=int, default=20, help="timed calls per size on the GPU")
    ap.add_argument("--warmup", type=int, default=3, help="warm-up calls per size and input kind")
    ap.add_argument("--cpu-iters", type=int, default=1, help="timed calls of the CPU oracle per size")
    ap.add_argument("--oracle-max", type=int, default=1024, help="largest size checked against the CPU oracle")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
