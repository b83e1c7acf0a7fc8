#!/usr/bin/env python
"""The HTTP API's terrain read-out (`GET /terrain?i1&j1&i2&j2&scale=`) after `get()`: upsample + crop + wire packing on the
device (`WorldPipeline.terrain_payload`) against the host path the reference runs on every request (api.py
`_get_terrain` + `_binary_response`: torch CPU `F.interpolate` of the whole padded native window, crop, numpy int16 pack
and channel interleave), on the same warm `get()` output.

    python tools/bench_terrain_api.py [--sizes 16,256,1024] [--scales 1,2,4,8] [--iters 50] [--cpu-iters 5] [--out FILE]

The pipeline has procedurally initialised models (bench.py's configurations); its tile cache is warmed with every
window first.  For each (size, scale) it prints, in one JSON line with the card's name and enforced power limit read in
the same run:
  device_ms          the read-out kernel per call: CUDA events around `iters` back-to-back launches;
  device_e2e_ms      kernel + the one pinned device->host copy + `bytes`, host clock;
  host_ms            the reference's host path on get()'s CPU tensors, host clock (torch CPU threads: all cores);
  request_device_ms  a whole warm `terrain_payload` call (its get() recomputes the elevation / climate read-out on
                     the device from cached tiles), host clock;
  request_host_ms    a warm `get()` of the padded window (CPU tensors out) + the host path, host clock;
  identical          the device body equals the host path's body byte for byte.
Writes nothing unless --out is given.
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


def power_limit_w(index: int):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        return None


def host_path(native: dict, scale: int, oi: int, oj: int, H: int, W: int) -> bytes:
    """What api.py does with get()'s CPU tensors: interpolate the whole padded window, crop, pack."""
    import numpy as np
    import torch.nn.functional as F
    elev, clim = native["elev"], native["climate"]
    if scale > 1:
        elev = F.interpolate(elev[None, None], scale_factor=scale, mode="bilinear", align_corners=False)[0, 0]
        clim = F.interpolate(clim[None], scale_factor=scale, mode="bilinear", align_corners=False)[0]
    elev, clim = elev[oi:oi + H, oj:oj + W], clim[:, oi:oi + H, oj:oj + W]
    e16 = np.clip(np.floor(elev.numpy().astype(np.float32, copy=False)), -32768, 32767).astype("<i2", copy=False)
    c = np.transpose(clim[:4].numpy().astype("<f4", copy=False), (1, 2, 0))
    return e16.tobytes() + c.tobytes()


def build_pipeline():
    import torch

    import bench as B
    from oracle import unet as ounet
    from terrain_diffusion_b200.inference import WorldPipeline
    from terrain_diffusion_b200.models import EDMUnet2D

    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m

    def cond_fn(i1, i2, j1, j2):
        gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0x7FFFFFFF)
        return torch.randn(5, i2 - i1, j2 - j1, generator=gg)

    pipe = WorldPipeline.from_local_models(build(B.COARSE_CFG), build(B.BASE_CFG), build(ounet.DECODER_CFG), seed=42,
                                           latents_batch_size=[1, 2, 4, 8, 16], cache_limit=None,
                                           conditioning_fn=cond_fn)
    return pipe.to("cuda").bind()


def run(args):
    import torch

    from terrain_diffusion_b200.inference import postproc
    if not torch.cuda.is_available():
        raise SystemExit("bench_terrain_api.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    pipe = build_pipeline()
    sizes = [int(s) for s in args.sizes.split(",")]
    scales = [int(s) for s in args.scales.split(",")]
    windows = [(n, s, (3, 5, 3 + n, 5 + n)) for n in sizes for s in scales]
    for _, s, w in windows:                                   # warm the tile cache with every native window
        pipe.terrain_payload(*w, scale=s)
    torch.cuda.synchronize()
    results = []
    for n, s, (i1, j1, i2, j2) in windows:
        ni1, nj1, ni2, nj2, oi, oj = postproc.terrain_window(i1, j1, i2, j2, s)
        native = pipe._get_device(ni1, nj1, ni2, nj2, True)
        native_cpu = {k: v.cpu() for k, v in native.items()}
        up = lambda: postproc.upsample_crop(native["elev"], native["climate"], s, oi, oj, n, n, payload=True)
        for _ in range(args.warmup):
            up()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            up()
        e1.record()
        torch.cuda.synchronize()
        device_ms = e0.elapsed_time(e1) / args.iters
        t0 = time.perf_counter()
        for _ in range(args.iters):
            body = postproc.to_host(up()).numpy().tobytes()
        e2e_ms = (time.perf_counter() - t0) * 1e3 / args.iters
        host_path(native_cpu, s, oi, oj, n, n)
        t0 = time.perf_counter()
        for _ in range(args.cpu_iters):
            ref = host_path(native_cpu, s, oi, oj, n, n)
        host_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters
        t0 = time.perf_counter()
        for _ in range(args.cpu_iters):
            pipe.terrain_payload(i1, j1, i2, j2, scale=s)
        req_dev_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters
        t0 = time.perf_counter()
        for _ in range(args.cpu_iters):
            host_path(pipe.get(ni1, nj1, ni2, nj2, with_climate=True), s, oi, oj, n, n)
        req_host_ms = (time.perf_counter() - t0) * 1e3 / args.cpu_iters
        results.append({"size": n, "scale": s, "native": [ni2 - ni1, nj2 - nj1], "device_ms": device_ms,
                        "device_e2e_ms": e2e_ms, "host_ms": host_ms, "speedup_e2e": host_ms / e2e_ms,
                        "request_device_ms": req_dev_ms, "request_host_ms": req_host_ms, "identical": body == ref})
        print(json.dumps(results[-1]), file=sys.stderr, flush=True)
    line = {"metric": "terrain API read-out after get(): upsample + crop + pack, per request", "unit": "ms",
            "iters": args.iters, "cpu_iters": args.cpu_iters, "warmup": args.warmup, "results": results,
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0)), "torch_threads": torch.get_num_threads(),
                     "torch": torch.__version__, "cpu_capability": torch.backends.cpu.get_cpu_capability()},
            "launches_per_call": 1}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="16,256,1024", help="comma-separated square request sizes (default: 16,256,1024)")
    ap.add_argument("--scales", default="1,2,4,8", help="comma-separated scales (default: 1,2,4,8)")
    ap.add_argument("--iters", type=int, default=50, help="timed device calls per case")
    ap.add_argument("--warmup", type=int, default=5, help="untimed device calls per case")
    ap.add_argument("--cpu-iters", type=int, default=5, help="timed host-path and whole-request calls per case")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
