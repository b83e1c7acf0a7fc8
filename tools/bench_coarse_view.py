#!/usr/bin/env python
"""The explorer's coarse map and the random sampler's land search on the device (`WorldPipeline.coarse_image`,
`coarse_data`, `coarse_stats`, `land_tiles`: kernels + one pinned copy) against the host path the reference runs on the
same canvas slice (server.py:58-185: one device->host copy of the slice per `_coarse_channel` call, then numpy; here the
oracle's restatement oracle/coarse_view.py; random_sampler.py:61-99: the Python double loop, restated on one host core).
PNG / JSON encoding is on the host in both and is not timed.

    python tools/bench_coarse_view.py [--sizes 100,600,2000] [--iters 50] [--cpu-iters 3] [--out FILE]

The canvas is a device tensor of seeded analytic (sum v*w, sum w) planes (tests/_coarse_view_inputs.py), so the numbers
measure the read-out, not the coarse diffusion.  For each (size, request) it prints, in one JSON line with the card's
name and enforced power limit read in the same run, medians of:
  device_ms      the launches alone, CUDA events around each call;
  device_e2e_ms  the whole method (launches + the pinned copy + the Python result), host clock;
  host_ms        the host path: the handler's slice copies (one per channel read) + numpy (+ `.tolist()` for
                 the data request, which the device path's result also includes), host clock;
  identical      the device result equals the host path's.
The land search (coarse_window 300, detail_size 1024, min_land_frac 0.5) is timed against the reference's loop restated
(`tile_land.mean().item()` per position on a CPU tensor, torch on one thread), over the first `--loop-rows` rows and
scaled to the whole window.  Writes profiles/bench_coarse_view.json unless --out says otherwise.
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

REQUESTS = ("image", "image_filtered", "data", "stats")
FILTERS = {0: (0.0, None), 2: (None, 18.0), 4: (100.0, None)}


def canvas_world(sums, origin: int):
    """A WorldPipeline whose coarse canvas is the device tensor `sums`, cell (0, 0) of it at (origin, origin)."""
    from terrain_diffusion_b200.inference.pipeline import WorldPipeline

    class CanvasWorld(WorldPipeline):
        def _coarse_sums(self, ci0, ci1, cj0, cj1):
            return sums[:, ci0 - origin:ci1 - origin, cj0 - origin:cj1 - origin]

    return CanvasWorld(native_resolution=90.0)


def host_call(request, sums, lut):
    """What the handler does with `world.coarse[...]`: each `_coarse_channel` call copies the slice to the host and
    divides; then numpy."""
    import numpy as np

    from oracle import coarse_view as O

    def read():
        return O.coarse_planes(sums.cpu().numpy())

    if request.startswith("image"):
        filters = FILTERS if request == "image_filtered" else {}
        planes = read()
        for _ in filters:                                                   # one more read per filter channel
            read()
        return O.coarse_image(planes, 4, lut, filters)[0]
    planes = np.stack([read()[c] for c in range(6)])
    if request == "stats":
        return O.coarse_stats(planes)
    return {"channels": {name: ch.tolist() for name, ch in zip(O.CHANNEL_NAMES, O.coarse_data(planes))}}


def device_call(world, request, win, lut):
    if request.startswith("image"):
        return world.coarse_image(*win, channel=4, filters=FILTERS if request == "image_filtered" else None, lut=lut)[0]
    if request == "data":
        return world.coarse_data(*win)
    return world.coarse_stats(*win)


def same(request, got, ref):
    import numpy as np
    if request.startswith("image"):
        return bool(np.array_equal(got, ref))
    if request == "data":
        return all(np.array_equal(np.array(got["channels"][n]), np.array(ref["channels"][n]), equal_nan=True)
                   for n in ref["channels"])
    return json.dumps(got, sort_keys=True) == json.dumps(ref, sort_keys=True)


def reference_loop_seconds(world_sums_host, cw, detail_size, min_land_frac, rows):
    """random_sampler.py:75-93 restated (the loop body unchanged) over the first `rows` rows; seconds per position."""
    import torch
    coarse = world_sums_host[:-1] / world_sums_host[-1:]
    coarse_elev_m = torch.sign(coarse[0]) * torch.square(coarse[0])
    land_mask = (coarse_elev_m > 0).float()
    H, W = land_mask.shape
    half = (detail_size // 256) // 2
    valid_tiles = []
    t0 = time.perf_counter()
    for i in range(half, half + rows):
        for j in range(half, W - half):
            tile_land = land_mask[i - half:i + half, j - half:j + half]
            if tile_land.mean().item() >= min_land_frac:
                valid_tiles.append((-cw + i, -cw + j))
    return (time.perf_counter() - t0) / (rows * (W - 2 * half)), valid_tiles


def run(args):
    import numpy as np
    import torch

    from bench_terrain_api import power_limit_w
    from oracle import coarse_view as O
    from tests._coarse_view_inputs import seeded_lut, world_sums
    if not torch.cuda.is_available():
        raise SystemExit("bench_coarse_view.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    lut = seeded_lut()
    results = []
    for n in [int(s) for s in args.sizes.split(",")]:
        lo = -(n // 2)
        sums = torch.from_numpy(world_sums("mixed", lo, lo + n, lo, lo + n)).to(dev)
        world = canvas_world(sums, lo)
        win = (lo, lo + n, lo, lo + n)
        for request in REQUESTS:
            call = lambda: device_call(world, request, win, lut)
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
                got = call()
                e2e_ms.append((time.perf_counter() - t0) * 1e3)
            host_ms = []
            for _ in range(args.cpu_iters):
                t0 = time.perf_counter()
                with np.errstate(invalid="ignore"):
                    ref = host_call(request, sums, lut)
                host_ms.append((time.perf_counter() - t0) * 1e3)
            entry = {"size": n, "request": request, "device_ms": statistics.median(dev_ms),
                     "device_e2e_ms": statistics.median(e2e_ms), "host_ms": statistics.median(host_ms)}
            entry["speedup_e2e"] = entry["host_ms"] / entry["device_e2e_ms"]
            entry["identical"] = same(request, got, ref)
            results.append(entry)
            print(json.dumps(entry), file=sys.stderr, flush=True)

    cw, detail, frac = 300, 1024, 0.5
    sums = torch.from_numpy(world_sums("mixed", -cw, cw, -cw, cw)).to(dev)
    world = canvas_world(sums, -cw)
    for _ in range(args.warmup):
        world.land_tiles(cw, detail, frac)
    land_ms = []
    for _ in range(args.iters):
        t0 = time.perf_counter()
        tiles = world.land_tiles(cw, detail, frac)
        land_ms.append((time.perf_counter() - t0) * 1e3)
    torch.set_num_threads(1)
    per_pos, loop_tiles = reference_loop_seconds(sums.cpu(), cw, detail, frac, args.loop_rows)
    half = (detail // 256) // 2
    positions = (2 * cw - 2 * half) ** 2
    want = O.land_tiles(sums.cpu().numpy(), -cw, -cw, detail, frac)
    land = {"coarse_window": cw, "detail_size": detail, "min_land_frac": frac, "positions": positions,
            "tiles": len(tiles), "device_e2e_ms": statistics.median(land_ms),
            "reference_loop_us_per_position": per_pos * 1e6, "reference_loop_rows_timed": args.loop_rows,
            "reference_loop_s_estimated": per_pos * positions,
            "identical": tiles == want and tiles[:len(loop_tiles)] == loop_tiles}
    land["speedup"] = land["reference_loop_s_estimated"] * 1e3 / land["device_e2e_ms"]
    print(json.dumps(land), file=sys.stderr, flush=True)
    line = {"metric": "explorer coarse map and sampler land search: per request", "unit": "ms",
            "statistic": "median", "iters": args.iters, "cpu_iters": args.cpu_iters, "warmup": args.warmup,
            "results": results, "land_search": land,
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0)), "numpy": np.__version__, "torch": torch.__version__}}
    text = json.dumps(line)
    print(text, flush=True)
    out = Path(args.out)
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="100,600,2000", help="comma-separated square window sizes in coarse cells "
                                                            "(default: 100,600,2000)")
    ap.add_argument("--iters", type=int, default=50, help="timed device calls per case (each way)")
    ap.add_argument("--warmup", type=int, default=5, help="untimed device calls per case")
    ap.add_argument("--cpu-iters", type=int, default=3, help="timed host-path calls per case")
    ap.add_argument("--loop-rows", type=int, default=20, help="rows of the reference's land loop timed (of 596)")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_coarse_view.json"), help="where the JSON line goes")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
