#!/usr/bin/env python
"""The Minecraft API's read-out (`mc-api` `GET /terrain?i1&j1&i2&j2&scale=&noise=`) after `get()`: upsample, Sobel
slope, detail noise, climate variables, biome classification and wire packing in one device launch
(`inference/minecraft.py` `readout`) against a host path on the same warm `get()` output and the same noise planes.

    python tools/bench_minecraft_api.py [--sizes 16,256,1024] [--scales 1,2,4,8] [--iters 50] [--cpu-iters 3] [--out FILE]

Noise generation is excluded from both sides: the five noise planes of each request are made once, before timing, and
handed to both.  The host path is the oracle's CPU restatement of the reference's (oracle/minecraft_api.py): torch CPU
`F.interpolate` of the whole padded native window and crop as the reference does, then the oracle's numpy Sobel,
climate variables and decision-list classifier (about 40 full-frame conditions instead of the reference's ~150 mask
writes) and the int16 packing.  It is a stand-in for the reference's host cost, not the reference itself.

For each (size, scale) it prints, in one JSON line with the card's name and enforced power limit read in the same run,
medians over the timed calls:
  device_ms      the read-out kernel per call: CUDA events around each launch;
  device_e2e_ms  kernel + the one pinned device->host copy + `bytes`, host clock;
  host_ms        the host path on get()'s CPU tensors, host clock (torch CPU threads: all cores);
  identical      the device body equals the host path's body byte for byte (it may differ at pixels within the
                 rounding bounds of tests/test_minecraft_gpu.py).
Writes nothing unless --out is given.
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
sys.path.insert(0, str(ROOT))


def power_limit_w(index: int):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        return None


def sm_clock_mhz(index: int):
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        return {"sm_now": pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM),
                "sm_max": pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)}
    except Exception:
        return None


def host_path(win, centre, climate, noise, scale, oi, oj, H, W, noise_scale, psm, nr) -> bytes:
    """The reference's host work on get()'s CPU tensors: whole-window torch bilinear upsample and crop (:288-317), then
    the oracle's Sobel, detail noise, climate variables and classifier, and the packing."""
    import numpy as np
    import torch.nn.functional as F

    from oracle import minecraft_api as O
    if scale > 1:
        up = F.interpolate(win[None, None], scale_factor=scale, mode="bilinear", align_corners=False)[0, 0]
        cl = F.interpolate(climate[None], scale_factor=scale, mode="bilinear", align_corners=False)[0]
        ring = up[oi - 1:oi + H + 1, oj - 1:oj + W + 1].numpy()
        cl = cl[:, oi:oi + H, oj:oj + W].numpy()
        r = O.readout(ring, cl, noise, 1, 1, 1, H, W, 0.0, psm, nr, centre=ring[1:-1, 1:-1])
        if noise_scale > 0:                    # the detail noise on the smooth elevation, as readout does above 1x
            g = r["vars"]["gradient"]
            sf = O._torch(lambda t: t.pow(1.5), O._clamp(g / np.float32(40.0 * psm / 90.0), 0.0, 1.0))
            ac = (np.float32(noise_scale * 100.0) * sf * np.float32(psm) / np.float32(nr)).astype(np.float32)
            af = (np.float32(noise_scale * 70.0) * sf * np.float32(psm) / np.float32(nr)).astype(np.float32)
            sm = r["elev_smooth"]
            r["elev"] = (sm + (noise[3] * ac + noise[4] * af) * (sm >= 0)).astype(np.float32)
    else:
        r = O.readout(win.numpy(), climate.numpy(), noise, 1, 1, 1, H, W, noise_scale, psm, nr, centre=centre.numpy())
    return O.payload(r["elev"], r["biome"])


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
    import numpy as np
    import torch

    from terrain_diffusion_b200.inference import minecraft as M
    from terrain_diffusion_b200.inference import postproc
    if not torch.cuda.is_available():
        raise SystemExit("bench_minecraft_api.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    pipe = build_pipeline()
    nr = float(pipe.native_resolution)
    sizes = [int(s) for s in args.sizes.split(",")]
    scales = [int(s) for s in args.scales.split(",")]
    results = []
    for n in sizes:
        for s in scales:
            i1, j1, i2, j2 = 3, 5, 3 + n, 5 + n
            wi1, wj1, wi2, wj2, oi, oj = M.minecraft_window(i1, j1, i2, j2, s)
            if s == 1:
                win = pipe._get_device(wi1, wj1, wi2, wj2, False)["elev"]
                native = pipe._get_device(i1, j1, i2, j2, True)
                centre, psm = native["elev"], nr
            else:
                native = pipe._get_device(wi1, wj1, wi2, wj2, True)
                win, centre, psm = native["elev"], None, nr / s
            rng = np.random.default_rng(n * 100 + s)
            noise = rng.uniform(-1, 1, (5, n, n)).astype(np.float32)     # made once: not part of either timing
            noise_d = torch.from_numpy(noise).to(dev)
            call = lambda: M.readout(win, native["climate"], noise_d, s, oi, oj, n, n, args.noise, psm, nr,
                                     centre=centre, payload=True)
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            ev = []
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                ev.append((e0, e1))
            torch.cuda.synchronize()
            device_ms = statistics.median(a.elapsed_time(b) for a, b in ev)
            e2e = []
            for _ in range(args.iters):
                t0 = time.perf_counter()
                body = postproc.to_host(call()).numpy().tobytes()
                e2e.append((time.perf_counter() - t0) * 1e3)
            cpu = [t.cpu() for t in (win, centre if centre is not None else win, native["climate"])]
            host_path(cpu[0], cpu[1], cpu[2], noise, s, oi, oj, n, n, args.noise, psm, nr)
            hs = []
            for _ in range(args.cpu_iters):
                t0 = time.perf_counter()
                ref = host_path(cpu[0], cpu[1], cpu[2], noise, s, oi, oj, n, n, args.noise, psm, nr)
                hs.append((time.perf_counter() - t0) * 1e3)
            r = {"size": n, "scale": s, "window": [wi2 - wi1, wj2 - wj1], "device_ms": device_ms,
                 "device_e2e_ms": statistics.median(e2e), "host_ms": statistics.median(hs),
                 "speedup_e2e": statistics.median(hs) / statistics.median(e2e), "identical": body == ref}
            results.append(r)
            print(json.dumps(r), file=sys.stderr, flush=True)
    line = {"metric": "Minecraft API read-out after get(): upsample + slope + detail noise + biomes + pack, per request",
            "unit": "ms", "statistic": "median", "noise": args.noise, "noise_generation": "excluded from both sides",
            "iters": args.iters, "cpu_iters": args.cpu_iters, "warmup": args.warmup, "results": results,
            "gpu": {"name": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(dev.index),
                    "clock_mhz": sm_clock_mhz(dev.index)},
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
    ap.add_argument("--noise", type=float, default=1.0, help="the request's noise parameter (default: 1.0)")
    ap.add_argument("--iters", type=int, default=50, help="timed device calls per case")
    ap.add_argument("--warmup", type=int, default=5, help="untimed device calls per case")
    ap.add_argument("--cpu-iters", type=int, default=3, help="timed host-path calls per case")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
