"""GPU bring-up of the wgmma implicit-GEMM conv: runs every case of tests/_igemm_ref.py, prints error statistics and,
on failure, a breakdown (by tile row/column, channel group, tap) that localises descriptor/layout mistakes.

Run on the GPU box:  python tools/bringup_igemm.py  (writes tool_out/bringup_igemm.txt as well)
"""
from __future__ import annotations

import os
import sys
import traceback

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from terrain_diffusion_b200 import _lib as L
from tests._igemm_ref import default_cases, make_inputs, plan_of, reference, rel_rms, run_cuda

LOG = []


def log(*a):
    s = " ".join(str(x) for x in a)
    print(s, flush=True)
    LOG.append(s)


def breakdown(got, ref):
    err = (got - ref).abs()
    bad = err > (0.02 * ref.abs() + 0.02)
    n, c, h, w = err.shape
    log("    bad fraction:", float(bad.float().mean()), " nan:", int(torch.isnan(got).sum()))
    by_y = bad.float().mean(dim=(0, 1, 3))
    by_x = bad.float().mean(dim=(0, 1, 2))
    by_c = bad.float().mean(dim=(0, 2, 3))
    log("    bad by row (first 18):", [round(float(v), 2) for v in by_y[:18]])
    log("    bad by col (first 18):", [round(float(v), 2) for v in by_x[:18]])
    log("    bad by channel (first 16):", [round(float(v), 2) for v in by_c[:16]])
    log("    got[0,0,:3,:6] =", got[0, 0, :3, :6].tolist())
    log("    ref[0,0,:3,:6] =", ref[0, 0, :3, :6].tolist())


def tap_probe(dev):
    """64->64 3x3 with weights only at one tap / one input channel: shows which tap / k-slice is mis-addressed."""
    import torch.nn.functional as F
    from terrain_diffusion_b200.layout import from_nc8hw8, pack_weight_segments, to_nc8hw8
    import ctypes as C
    g = torch.Generator().manual_seed(1)
    a = torch.randn(1, 64, 16, 8, generator=g).bfloat16().float().to(dev)
    for tap in range(9):
        for kch in (0, 9, 17, 63):
            w = torch.zeros(64, 64, 3, 3, device=dev)
            for n in range(64):
                w[n, kch, tap // 3, tap % 3] = 1.0 + n / 64.0
            ref = F.conv2d(a, w, padding=1)
            d = L.TdxIgemmDesc()
            an = to_nc8hw8(a)
            b = pack_weight_segments([w]).to(dev)
            o = torch.full((1, 8, 16, 8, 8), float("nan"), dtype=torch.bfloat16, device=dev)
            d.a_ptr[0] = an.data_ptr(); d.a_channels[0] = 64; d.a_taps[0] = 9; d.n_seg = 1
            d.b_packed = b.data_ptr(); d.c_out = 64; d.n_per_item = 64; d.n_img = 1; d.height = 16; d.width = 8
            d.out[0].ptr = o.data_ptr(); d.out[0].kind = L.OUT_RAW; d.out[0].spatial = L.SP_SAME; d.out[0].scale = 1.0
            L.check(L.lib().tdx_igemm_run(C.byref(d), L.current_stream_ptr()))
            torch.cuda.synchronize()
            got = from_nc8hw8(o)
            e = float((got - ref.bfloat16().float()).abs().max())
            if e > 0.05:
                log(f"  tap_probe tap={tap} kch={kch}: max err {e:.4f}")
                log("    got[0,0,:4,:8] =", got[0, 0, :4, :8].tolist())
                log("    ref[0,0,:4,:8] =", ref[0, 0, :4, :8].tolist())
                return False
    log("  tap_probe: all taps / k-slices exact")
    return True


def main():
    dev = torch.device("cuda:0")
    log("device:", torch.cuda.get_device_name(0))
    import ctypes as C
    sm, ma, mi = C.c_int(), C.c_int(), C.c_int()
    L.check(L.lib().tdx_device_info(C.byref(sm), C.byref(ma), C.byref(mi)))
    log(f"sm_count={sm.value} cc={ma.value}.{mi.value}")
    n_fail = 0
    try:
        ok = tap_probe(dev)
        n_fail += 0 if ok else 1
    except Exception:
        log("tap_probe raised:\n" + traceback.format_exc())
        n_fail += 1
    for case in default_cases():
        try:
            acts, wts, cvec, resid = make_inputs(case, dev)
            plan = plan_of(case)
            log(f"     plan {case.name}: N={plan['N']} ksplit={plan['ks']} resident={plan['resident']} SB={plan['SB']} "
                f"cluster={plan['cluster']} rounds={plan['rounds']}")
            refs = reference(case, acts, wts, cvec, resid)
            gots = run_cuda(case, acts, wts, cvec, resid)
            worst = 0.0
            for i, (g_, r_) in enumerate(zip(gots, refs)):
                rr = rel_rms(g_, r_.bfloat16().float())
                mx = float((g_ - r_).abs().max())
                worst = max(worst, rr)
                status = "ok " if rr < 1e-2 and not torch.isnan(g_).any() else "BAD"
                log(f"[{status}] {case.name} out{i}: rel_rms={rr:.3e} max_abs={mx:.3e}")
                if status == "BAD":
                    breakdown(g_, r_)
                    n_fail += 1
        except Exception:
            log(f"[EXC] {case.name}:\n" + traceback.format_exc())
            n_fail += 1
            if "CUDA" in traceback.format_exc() or "cuda" in traceback.format_exc():
                break
    log("FAILURES:", n_fail)
    os.makedirs("tool_out", exist_ok=True)
    with open("tool_out/bringup_igemm.txt", "w") as f:
        f.write("\n".join(LOG) + "\n")
    return 1 if n_fail else 0


if __name__ == "__main__":
    sys.exit(main())
