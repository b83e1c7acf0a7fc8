"""Micro-benchmark of the wgmma implicit-GEMM conv on the decoder's layer shapes (CUDA events, L2 flushed).

Run on the GPU box:  python tools/bench_igemm.py [--batch N]   -> tool_out/bench_igemm.txt
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.layout import pack_weight_segments, to_nc8hw8

# (name, segs [(C, taps)], cout, res-at-256-input, count per forward)
SHAPES = [
    ("64->64 3x3 @256", [(64, 9)], 64, 256, 10),
    ("128->64 (concat) 3x3 @256", [(64, 9), (64, 9)], 64, 256, 3),
    ("res1+skip 64*9+128 ->64 @256", [(64, 9), (64, 1), (64, 1)], 64, 256, 3),
    ("128->128 3x3 @256 (up)", [(128, 9)], 128, 256, 2),
    ("128->128 3x3 @128", [(128, 9)], 128, 128, 10),
    ("256->128 (concat) 3x3 @128", [(128, 9), (128, 9)], 128, 128, 2),
    ("192->192 3x3 @128 (up)", [(192, 9)], 192, 128, 2),
    ("192->192 3x3 @64", [(192, 9)], 192, 64, 10),
    ("384->192 (concat) 3x3 @64", [(192, 9), (192, 9)], 192, 64, 2),
    ("256->256 3x3 @64 (up)", [(256, 9)], 256, 64, 2),
    ("256->256 3x3 @32", [(256, 9)], 256, 32, 14),
    ("512->256 (concat) 3x3 @32", [(256, 9), (256, 9)], 256, 32, 3),
    ("64->128 1x1 @128", [(64, 1)], 128, 128, 1),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lines = []
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    tot_t, tot_f = 0.0, 0.0
    for name, segs, cout, res, count in SHAPES:
        n = args.batch
        acts = [to_nc8hw8(torch.randn(n, c, res, res, device=dev)) for c, _ in segs]
        wts = [torch.randn(cout, c, 3 if t == 9 else 1, 3 if t == 9 else 1, device=dev) * 0.02 for c, t in segs]
        n_item = L.igemm_choose_n(cout, n, res, res, segs)
        b = pack_weight_segments(wts, n_item)
        out = torch.empty(n, cout // 8, res, res, 8, dtype=torch.bfloat16, device=dev)
        d = L.TdxIgemmDesc()
        for i, (c, t) in enumerate(segs):
            d.a_ptr[i] = acts[i].data_ptr(); d.a_channels[i] = c; d.a_taps[i] = t
        d.n_seg = len(segs); d.b_packed = b.data_ptr(); d.c_out = cout; d.n_per_item = n_item
        d.n_img, d.height, d.width = n, res, res
        d.out[0].ptr = out.data_ptr(); d.out[0].kind = L.OUT_RAW; d.out[0].scale = 1.0
        stream = L.current_stream_ptr()
        for _ in range(3):
            L.check(L.lib().tdx_igemm_run(C.byref(d), stream))
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.iters):
            flush.zero_()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            L.check(L.lib().tdx_igemm_run(C.byref(d), stream))
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        ms = ts[len(ts) // 2]
        flops = 2.0 * n * res * res * cout * sum(c * t for c, t in segs)
        tf = flops / ms / 1e9
        tot_t += ms * count
        tot_f += flops * count
        s = f"{name:34s} N={n} {ms*1e3:9.1f} us  {tf:8.1f} TFLOP/s  (x{count}/fwd, min {ts[0]*1e3:.1f} us)"
        print(s, flush=True)
        lines.append(s)
    s = f"weighted: {tot_t:.3f} ms per forward-equivalent, {tot_f/tot_t/1e9:.1f} TFLOP/s"
    print(s)
    lines.append(s)
    os.makedirs("tool_out", exist_ok=True)
    with open(f"tool_out/bench_igemm_b{args.batch}.txt", "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
