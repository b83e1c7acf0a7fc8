"""Achieved HBM bandwidth of the memory-bound kernels of the path (blend, normalise, scheduler step, im2col, conv_out)
and the generation rate of the tile noise, against the measured copy bandwidth in MEASURED_PEAKS.json when it exists,
else against the 3 350 GB/s of HBM3 the H100 SXM data sheet rates (a rated figure, not a measured one).
Algorithmic bytes per launch (what must cross HBM once) / CUDA-event time, L2 flushed between launches.

    python tools/bench_hbm_kernels.py > tool_out/hbm_kernels.txt
"""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference.noise import gaussian_noise_patch
from terrain_diffusion_b200.inference.tiling import linear_weight_window

dev = torch.device("cuda:0")
lib = L.lib()
peak, peak_name = 3350.0, "H100 SXM data-sheet HBM3 bandwidth"
try:
    peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
    peak_name = "measured copy peak"
except Exception:
    pass
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, reps=10):
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def report(name, nbytes, ms):
    gbs = nbytes / (ms * 1e-3) / 1e9
    print(f"{name:58s} {nbytes / 1e6:9.1f} MB  {ms * 1e3:8.1f} us  {gbs:8.1f} GB/s  {gbs / peak:5.2f} of {peak_name}")


s = L.current_stream_ptr()
for T, Ccv in ((512, 1), (512, 5), (64, 6)):
    H = 4096
    val = torch.zeros(Ccv, H, H, device=dev); ws = torch.zeros(H, H, device=dev)
    tile = torch.randn(Ccv, T, T, device=dev); win = linear_weight_window(T, dev).contiguous()
    n = 16
    def f():
        for k in range(n):
            lib.tdx_blend_accumulate(val.data_ptr(), ws.data_ptr(), Ccv, H, H, tile.data_ptr(), win.data_ptr(), T, T,
                                     (k % 4) * 384 * (T // 64) // 8 * 8, (k // 4) * 384 * (T // 64) // 8 * 8, s)
    ms = timeit(f) / n
    report(f"blend_accumulate tile {T}^2 x {Ccv} ch (float4)", (Ccv * 3 + 3) * T * T * 4, ms)
H = 8192
val = torch.randn(1, H, H, device=dev); ws = torch.rand(H, H, device=dev) + 0.5; out = torch.empty_like(val)
ms = timeit(lambda: lib.tdx_blend_normalize(out.data_ptr(), val.data_ptr(), ws.data_ptr(), 1, H * H, 0.5, s))
report("blend_normalize 8192^2 x 1 ch (float4)", 3 * H * H * 4, ms)
n = 16 * 256 * 256
a, b, c = (torch.randn(n, device=dev) for _ in range(3))
ms = timeit(lambda: lib.tdx_sched_step(a.data_ptr(), b.data_ptr(), c.data_ptr(), n, 0.3, 0.4, 0.5, 0.1, s))
report("sched_step 16 x 256^2 (3 reads + 2 writes)", 5 * n * 4, ms)
# im2col + conv_out on 16 tiles of 256^2
N, S = 16, 256
x1 = torch.randn(N, 1, S, S, device=dev); x2 = torch.randn(N, 4, S, S, device=dev)
cols = torch.empty(N, 8, S, S, 8, dtype=torch.bfloat16, device=dev)
im = L.TdxIm2colDesc()
im.src[0], im.src[1] = x1.data_ptr(), x2.data_ptr(); im.src_channels[0], im.src_channels[1] = 1, 4
im.out = cols.data_ptr(); im.k_pad = 64; im.n_img, im.height, im.width = N, S, S
ms = timeit(lambda: L.check(lib.tdx_im2col_run(C.byref(im), s)))
report("im2col 16 x 256^2 (5 fp32 planes in, 64 bf16 'channels' out)", N * S * S * (5 * 4 + 128), ms)
xin = torch.randn(N, 8, S, S, 8, device=dev).bfloat16(); wgt = torch.randn(9, 64, 1, device=dev)
mo = torch.empty(N, 1, S, S, device=dev)
od = L.TdxConvOutDesc()
od.x = xin.data_ptr(); od.c_in = 64; od.weight = wgt.data_ptr(); od.c_out = 1; od.n_img, od.height, od.width = N, S, S
od.model_out = mo.data_ptr()
ms = timeit(lambda: L.check(lib.tdx_conv_out_run(C.byref(od), s)))
report("conv_out 16 x 256^2 (64 bf16 channels in, 1 fp32 plane out)", N * S * S * (128 + 4), ms)
ms = timeit(lambda: gaussian_noise_patch(1234, 384, -384, 512, 512, 1, 512, 512, device=dev))
print(f"{'tile noise 512^2 x 1 ch (PCG + polar, bit-exact stream)':58s} {512 * 512 / (ms * 1e-3) / 1e6:9.1f} M normals/s  "
      f"{ms * 1e3:8.1f} us per tile (integer / fp64 bound, not HBM)")
