"""Per-tile phase timeline of CTA 0 of the igemm kernel (debug hook tdx_debug_set_igemm_trace).

    python tools/trace_igemm.py              # phase clocks of a few launch shapes
    python tools/trace_igemm.py floor        # launch floor of an empty-ish kernel
"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
# the hooks this tool reads are compiled out of the production kernel: (re)build libtdx.so with them
# (run `python -m terrain_diffusion_b200.build` afterwards to get the production library back)
os.environ["TDX_DEBUG_HOOKS"] = "1"
from terrain_diffusion_b200.build import build as _build  # noqa: E402
import importlib, terrain_diffusion_b200.build as _b  # noqa: E402
importlib.reload(_b).build()
import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.layout import pack_weight_segments, to_nc8hw8

SHAPES = [("64->64 1x1 @16 (tiny)", [(64, 1)], 64, 16), ("64->64 @128 (<=2 items/CTA)", [(64, 9)], 64, 128), ("64->64 @256", [(64, 9)], 64, 256), ("128->128 @128", [(128, 9)], 128, 128),
          ("256->256 @32", [(256, 9)], 256, 32), ("192->192 @64", [(192, 9)], 192, 64)]
NAMES = ["A-prod start", "mma: start", "mma: acc staged", "split-K: partials published", "epi: done"]


def main():
    dev = torch.device("cuda:0")
    lib = L.lib()
    lib.tdx_debug_set_igemm_trace.argtypes = [C.c_void_p]
    trace = torch.zeros(128, dtype=torch.int64, device=dev)
    for name, segs, cout, res in SHAPES + [("RES1 64->64 @256 (resid pnorm, 3 outputs)", [(64, 9)], 64, 256)]:
        acts = [to_nc8hw8(torch.randn(1, c, res, res, device=dev)) for c, _ in segs]
        wts = [torch.randn(cout, c, 3, 3, device=dev) * 0.02 for c, t in segs]
        n_item = L.igemm_choose_n(cout, 1, res, res, segs)
        b = pack_weight_segments(wts, n_item)
        out = torch.empty(1, cout // 8, res, res, 8, dtype=torch.bfloat16, device=dev)
        cvec = torch.ones(1, cout, device=dev)
        d = L.TdxIgemmDesc()
        for i, (c, t) in enumerate(segs):
            d.a_ptr[i] = acts[i].data_ptr(); d.a_channels[i] = c; d.a_taps[i] = t
        d.n_seg = len(segs); d.b_packed = b.data_ptr(); d.c_out = cout; d.n_per_item = n_item
        d.n_img, d.height, d.width = 1, res, res
        d.epi_flags = L.EPI_EMB_SILU; d.cvec = cvec.data_ptr()
        d.out[0].ptr = out.data_ptr(); d.out[0].kind = L.OUT_RAW; d.out[0].scale = 1.0
        if name.startswith("RES1"):
            resid = to_nc8hw8(torch.randn(1, cout, res, res, device=dev))
            out2 = torch.empty_like(out); out3 = torch.empty_like(out)
            d.epi_flags = L.EPI_RESID; d.resid = resid.data_ptr(); d.resid_pnorm = 1; d.resid_scale = 0.9; d.clip = 256.0
            d.out[1].ptr = out2.data_ptr(); d.out[1].kind = L.OUT_PNORM_SILU; d.out[1].scale = 1.0
            d.out[2].ptr = out3.data_ptr(); d.out[2].kind = L.OUT_SILU; d.out[2].scale = 0.8
        for _ in range(2):
            L.check(lib.tdx_igemm_run(C.byref(d), L.current_stream_ptr()))
        torch.cuda.synchronize()
        trace.zero_()
        lib.tdx_debug_set_igemm_trace(trace.data_ptr())
        L.check(lib.tdx_igemm_run(C.byref(d), L.current_stream_ptr()))
        torch.cuda.synchronize()
        lib.tdx_debug_set_igemm_trace(None)
        t = trace.cpu().tolist()
        t0 = t[127]
        print(f"== {name}: clocks relative to CTA-0 setup done; kernel entry at {t[126]-t0}, exit at {t[125]-t0}")
        for it in range(4):
            row = t[it * 8: it * 8 + len(NAMES)]
            if row[0] == 0 and row[1] == 0:
                break
            print(f"  tile {it}: " + "  ".join(f"{n}={v - t0 if v else -1}" for n, v in zip(NAMES, row)))


def launch_floor():
    """Average time per launch of a tiny igemm inside a 200-launch program replayed as a graph."""
    from terrain_diffusion_b200.models.plan import UNetProgram
    dev = torch.device("cuda:0")
    for name, segs, cout, res in [("tiny 1x1 16x16", [(64, 1)], 64, 16), ("64->64 3x3 @32 (8 items)", [(64, 9)], 64, 32),
                                  ("64->64 3x3 @256", [(64, 9)], 64, 256)]:
        acts = [to_nc8hw8(torch.randn(1, c, res, res, device=dev)) for c, _ in segs]
        wts = [torch.randn(cout, c, 3 if t == 9 else 1, 3 if t == 9 else 1, device=dev) * 0.02 for c, t in segs]
        n_item = L.igemm_choose_n(cout, 1, res, res, segs)
        b = pack_weight_segments(wts, n_item)
        outs = [torch.empty(1, cout // 8, res, res, 8, dtype=torch.bfloat16, device=dev) for _ in range(2)]
        prog = UNetProgram()
        for i in range(200):
            d = L.TdxIgemmDesc()
            src = acts[0] if i == 0 else outs[(i + 1) % 2]
            d.a_ptr[0] = src.data_ptr(); d.a_channels[0] = segs[0][0]; d.a_taps[0] = segs[0][1]
            d.n_seg = 1; d.b_packed = b.data_ptr(); d.c_out = cout; d.n_per_item = n_item
            d.n_img, d.height, d.width = 1, res, res
            d.out[0].ptr = outs[i % 2].data_ptr(); d.out[0].kind = L.OUT_RAW; d.out[0].scale = 1.0
            L.check(L.lib().tdx_program_add_igemm(prog.handle, C.byref(d)))
        prog.keep += [acts, b, outs]
        for _ in range(3):
            prog.run(True)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            prog.run(True)
        e1.record()
        torch.cuda.synchronize()
        print(f"launch floor [{name}]: {e0.elapsed_time(e1) / 1000 * 1e3:.2f} us per dependent launch (graph)")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "floor":
        launch_floor()
        sys.exit(0)
    main()
