#!/usr/bin/env python
"""The explorer's detail view after `get()`: the `/api/detail.png` pictures (modes elevation, temperature, relief) and
the `/api/detail_raw` body, on the device (`WorldPipeline.get_detail` / `detail_raw_payload`: kernels + one pinned copy)
against the host path the reference's handlers run (server.py:188-270: `world.get()`'s copy of the elevation and all
five climate planes, then numpy / matplotlib on the host, here the oracle's restatement oracle/explorer.py, and for the
relief oracle/relief.py), on the same warm `get()` output.  PNG encoding is on the host in both and is not timed.

    python tools/bench_explorer.py [--sizes 512,1024,2048] [--iters 50] [--cpu-iters 3] [--out FILE]

The pipeline has procedurally initialised models (bench.py's configurations); its tile cache is warmed with every
window first, so the numbers measure the read-out, not diffusion.  For each (size, mode) it prints, in one JSON line with
the card's name and enforced power limit read in the same run, medians of:
  device_ms      the launches alone, CUDA events around each call (relief: the four relief launches included);
  device_e2e_ms  the launches + the one pinned device->host copy (+ `bytes` for raw), host clock;
  host_ms        get()'s device->host copy of elevation + 5 climate planes, then the host steps, host clock;
  identical      the device result equals the host path's (relief: `relief_px_differ` counts the pixels that differ,
                 from the relief's colormap-boundary pixels, DESIGN.md section 4.4).
Writes profiles/bench_explorer.json unless --out says otherwise.
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

MODES = ("elevation", "temperature", "relief", "raw")


def device_call(mode, elev, climate, native_resolution):
    """The device work of one request on get()'s device planes; returns the CUDA result."""
    from terrain_diffusion_b200.inference import explorer as E
    from terrain_diffusion_b200.inference.relief import get_relief_map
    if mode == "elevation":
        return E.colour_image(elev, "terrain")
    if mode == "temperature":
        return E.colour_image(climate[0], "RdBu_r")
    if mode == "relief":
        return E.relief_rgba8(get_relief_map(elev, None, None, None, resolution=native_resolution))
    return E.raw_body(elev, climate[0])


def host_call(mode, elev, climate, native_resolution):
    """What the handler does after `world.get()`: the copy to the host, then numpy (oracle restatement)."""
    import numpy as np

    from oracle import explorer as O
    e, c = elev.cpu().numpy(), climate.cpu().numpy()
    if mode == "raw":
        return O.detail_raw_body(e, c[0])
    with np.errstate(invalid="ignore"):
        return O.detail_image(e, c[0], mode, native_resolution)


def run(args):
    import numpy as np
    import torch

    from bench_terrain_api import build_pipeline, power_limit_w
    from terrain_diffusion_b200.inference import postproc
    if not torch.cuda.is_available():
        raise SystemExit("bench_explorer.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    pipe = build_pipeline()
    sizes = [int(s) for s in args.sizes.split(",")]
    windows = {n: (3, 5, 3 + n, 5 + n) for n in sizes}
    for w in windows.values():                                # warm the tile cache with every window
        pipe.get_detail(*w, mode="temperature")
    torch.cuda.synchronize()
    res = pipe.native_resolution
    results = []
    for n, w in windows.items():
        native = pipe._get_device(*w, True)
        elev, climate = native["elev"], native["climate"]
        for mode in MODES:
            call = lambda: device_call(mode, elev, climate, res)
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            dev_ms, e2e_ms = [], []
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                e1.synchronize()
                dev_ms.append(e0.elapsed_time(e1))
            for _ in range(args.iters):
                t0 = time.perf_counter()
                got = postproc.to_host(call()).numpy()
                if mode == "raw":
                    got = got.tobytes()
                e2e_ms.append((time.perf_counter() - t0) * 1e3)
            host_ms = []
            for _ in range(args.cpu_iters):
                t0 = time.perf_counter()
                ref = host_call(mode, elev, climate, res)
                host_ms.append((time.perf_counter() - t0) * 1e3)
            entry = {"size": n, "mode": mode, "device_ms": statistics.median(dev_ms),
                     "device_e2e_ms": statistics.median(e2e_ms), "host_ms": statistics.median(host_ms)}
            entry["speedup_e2e"] = entry["host_ms"] / entry["device_e2e_ms"]
            if mode == "raw":
                entry["identical"] = got == ref
            else:
                differ = int((got != ref).any(axis=-1).sum())
                entry["identical"] = differ == 0
                if mode == "relief":
                    entry["relief_px_differ"] = differ
            results.append(entry)
            print(json.dumps(entry), file=sys.stderr, flush=True)
    line = {"metric": "explorer detail view after get(): image / raw body per request", "unit": "ms",
            "statistic": "median", "iters": args.iters, "cpu_iters": args.cpu_iters, "warmup": args.warmup,
            "results": results,
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0)), "numpy": np.__version__, "torch": torch.__version__}}
    text = json.dumps(line)
    print(text, flush=True)
    out = Path(args.out)
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="512,1024,2048", help="comma-separated square window sizes (default: "
                                                              "512,1024,2048)")
    ap.add_argument("--iters", type=int, default=50, help="timed device calls per case (each way)")
    ap.add_argument("--warmup", type=int, default=5, help="untimed device calls per case")
    ap.add_argument("--cpu-iters", type=int, default=3, help="timed host-path calls per case")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_explorer.json"), help="where the JSON line goes")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
