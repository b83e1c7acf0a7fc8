"""The fp32 glue kernels every sampler and pipeline stage runs between the U-Net launches, each through its C entry
point against a plain fp32 restatement on the CPU that rounds once per operation in the kernel's order: the overlap
blend (tdx_blend_accumulate, tdx_blend_normalize), the DPM-Solver++ update (tdx_sched_step), the consistency-stage glue
(tdx_trig_mix, tdx_pack_weighted, tdx_window_to_cond) and the raw normal stream (tdx_standard_normal).

Every kernel promises bit-identical results (explicitly rounded __fmul_rn / __fadd_rn / __fdiv_rn, no contraction), so
every comparison is on bit patterns: -0.0 and +0.0 differ, and NaN must appear in exactly the reference's positions
(payloads differ between CUDA and x86, so only positions are compared).  Each case is named after the path it takes
through its kernel -- float4 interior, float4 edge, scalar, or grid-stride (more elements than one pass of the capped
grid covers; the test asserts the count really is above the cap on this device).  Every output lives in a guarded
buffer (tests/_igemm_ref.Guarded): a write outside the tensor fails."""
from __future__ import annotations

import math
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import rng as orng
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference.canvas import BlendCanvas
from terrain_diffusion_b200.inference.noise import MASK64, standard_normal
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests._igemm_ref import SENTINEL32, Guarded
from tests.test_direct_kernels_gpu import _sched_update_fp32

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = torch.float32
G = np.load(Path(__file__).resolve().parent / "golden" / "reference_golden.npz")


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


class _Buf:
    """fp32 `shape` inside a Guarded allocation, starting `offset` elements past its 16-byte-aligned start (offset 1
    gives a pointer that is 4- but not 16-byte aligned, which sends the launch to a kernel's scalar path).  The
    skipped lead elements hold the sentinel too and are checked with the guards."""

    def __init__(self, shape, init: torch.Tensor | None = None, offset: int = 0):
        shape = tuple(shape)
        self.offset = offset
        self.g = Guarded((offset + math.prod(shape),), F32, DEV)
        self.g.view[:offset].view(torch.int32).fill_(SENTINEL32)
        self.view = self.g.view[offset:].view(shape)
        if init is not None:
            self.view.copy_(init)

    def ptr(self) -> int:
        return self.view.data_ptr()

    def check(self, what: str):
        torch.cuda.synchronize()
        self.g.check(what)
        lead = self.g.view[:self.offset].view(torch.int32)
        assert bool((lead == SENTINEL32).all()), f"{what}: written before the tensor's first element"


def _launch(fn, *args):
    L.call(fn, DEV, *args)
    torch.cuda.synchronize()


def assert_bits(got: torch.Tensor, want: torch.Tensor, what: str):
    """Bit-identical wherever `want` is not NaN; NaN in exactly the same positions."""
    got, want = got.detach().cpu().contiguous(), want.detach().cpu().contiguous()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan_g, nan_w = torch.isnan(got), torch.isnan(want)
    assert torch.equal(nan_g, nan_w), f"{what}: NaN positions differ at {int((nan_g ^ nan_w).sum())} elements"
    diff = (got.view(torch.int32) != want.view(torch.int32)) & ~nan_w
    n = int(diff.sum())
    if n:
        i = tuple(int(v) for v in diff.nonzero()[0])
        raise AssertionError(f"{what}: {n} of {int((~nan_w).sum())} elements differ in their bits; first at {i}: "
                             f"got {float(got[i])!r}, want {float(want[i])!r}")


def _f32(v: float) -> torch.Tensor:
    """A scalar as the fp32 value the C entry point receives (ctypes rounds a double to the nearest float)."""
    return torch.tensor(v, dtype=F32)


def _window(g, th: int, tw: int) -> torch.Tensor:
    """Random positive blend weights with about one in ten exactly zero."""
    w = torch.rand(th, tw, generator=g) + 0.05
    w[torch.rand(th, tw, generator=g) < 0.1] = 0.0
    return w


# ------------------------------------------------------------------------------------------------ blend_accumulate
def _accumulate_ref(val, wsum, tile, win, y0, x0):
    """oracle/tiling.accumulate (val += tile * w ; wsum += w), clipped to the canvas: a tile may hang over any edge."""
    _, ch, cw = val.shape
    th, tw = win.shape
    ya, yb, xa, xb = max(y0, 0), min(y0 + th, ch), max(x0, 0), min(x0 + tw, cw)
    if ya >= yb or xa >= xb:
        return
    w = win[ya - y0:yb - y0, xa - x0:xb - x0]
    val[:, ya:yb, xa:xb] += tile[:, ya - y0:yb - y0, xa - x0:xb - x0] * w
    wsum[ya:yb, xa:xb] += w


def _blend_scalar_clauses(ch, cw, th, tw, x0, ptrs) -> set:
    """The clauses of tdx_blend_accumulate's float4 predicate that this launch fails (empty: the float4 kernel)."""
    failed = set()
    if tw % 4:
        failed.add("tile_w")
    if cw % 4:
        failed.add("canvas_w")
    if x0 % 4:
        failed.add("x0")
    if any(p % 16 for p in ptrs):
        failed.add("pointer")
    if (ch * cw) % 4 or (th * tw) % 4:
        failed.add("plane")
    return failed


# name: (canvas h, w, tile h, w, canvas origins of the tiles in replay order, canvas pointer offset in floats,
#        the float4 clause every launch fails)
BLEND_CASES = {
    "float4-interior": (100, 148, 40, 64, [(0, 0), (0, 44), (30, 20), (36, 84), (60, 84)], 0, None),
    "float4-left-edge-x0=-8": (100, 148, 40, 64, [(10, -8), (30, -8), (20, 0), (0, -8)], 0, None),
    "float4-clipped-top-bottom": (100, 148, 40, 64, [(-10, 8), (-25, 40), (70, 8), (85, 80), (-39, 84)], 0, None),
    "float4-outside-every-side": (100, 148, 40, 64, [(-40, 0), (100, 0), (0, -64), (0, 148), (-40, -64),
                                                     (100, 148), (-400, 4), (4, 1000)], 0, None),
    "float4-tile-larger-than-canvas": (24, 32, 40, 64, [(-8, -16), (-12, -20), (-16, -32)], 0, None),
    "scalar-tile_w=37": (100, 148, 40, 37, [(0, 0), (10, 40), (70, 112), (-5, -8), (20, 120)], 0, "tile_w"),
    "scalar-canvas_w=150": (100, 150, 40, 64, [(0, 0), (20, 44), (60, 88), (30, 100), (-12, -4)], 0, "canvas_w"),
    "scalar-x0=5": (100, 148, 40, 64, [(0, 5), (30, 5), (60, 5), (-10, 5)], 0, "x0"),
    "scalar-x0=85": (100, 148, 40, 64, [(0, 85), (30, 85), (75, 85)], 0, "x0"),
    "scalar-x0=-6": (100, 148, 40, 64, [(0, -6), (30, -6), (10, -6), (75, -6)], 0, "x0"),
    "scalar-canvas-pointer+1": (100, 148, 40, 64, [(0, 0), (0, 44), (30, 20), (-10, -8), (70, 88), (36, 84)], 1,
                                "pointer"),
}


def _run_blend(ch, cw, th, tw, origins, channels, seed, val_offset=0, wsum_offset=0):
    """Replays `origins` onto a non-zero canvas through tdx_blend_accumulate and through _accumulate_ref; returns
    (device val, device wsum, reference val, reference wsum, the float4 clauses each launch failed)."""
    g = torch.Generator().manual_seed(seed)
    win = _window(g, th, tw)
    val0 = torch.randn(channels, ch, cw, generator=g) * 4
    wsum0 = torch.rand(ch, cw, generator=g) * 2
    val, wsum = _Buf(val0.shape, val0, val_offset), _Buf(wsum0.shape, wsum0, wsum_offset)
    win_d = win.to(DEV)
    ref_v, ref_w = val0.clone(), wsum0.clone()
    clauses = []
    for y0, x0 in origins:
        tile = torch.randn(channels, th, tw, generator=g) * 3
        tile_d = tile.to(DEV)
        clauses.append(_blend_scalar_clauses(ch, cw, th, tw, x0,
                                             (val.ptr(), wsum.ptr(), tile_d.data_ptr(), win_d.data_ptr())))
        _launch(L.lib().tdx_blend_accumulate, val.ptr(), wsum.ptr(), channels, ch, cw, tile_d.data_ptr(),
                win_d.data_ptr(), th, tw, y0, x0)
        val.check(f"val after the tile at {(y0, x0)}")
        wsum.check(f"wsum after the tile at {(y0, x0)}")
        _accumulate_ref(ref_v, ref_w, tile, win, y0, x0)
    return val.view.cpu(), wsum.view.cpu(), ref_v, ref_w, clauses


@pytest.mark.parametrize("channels", [1, 3, 18])
@pytest.mark.parametrize("case", list(BLEND_CASES))
def test_blend_accumulate(case, channels):
    ch, cw, th, tw, origins, offset, clause = BLEND_CASES[case]
    got_v, got_w, ref_v, ref_w, clauses = _run_blend(ch, cw, th, tw, origins, channels, seed=len(case) * 7 + channels,
                                                     val_offset=offset)
    want = set() if clause is None else {clause}
    assert all(c == want for c in clauses), clauses            # exactly the named clause sends it to the scalar kernel
    assert_bits(got_v, ref_v, f"{case} val")
    assert_bits(got_w, ref_w, f"{case} wsum")


@pytest.mark.parametrize("channels", [1, 3, 18])
def test_blend_accumulate_float4_and_scalar_kernels_are_bit_identical(channels):
    """One tile sequence (interior, edges, overhangs) on an aligned canvas (float4 kernel) and on one whose planes start
    one float later (scalar kernel): both equal the reference and each other bit for bit."""
    args = (100, 148, 40, 64, [(0, 0), (-10, -8), (30, 44), (70, 88), (85, 100), (20, 140), (-30, 120)], channels)
    v4, w4, ref_v, ref_w, c4 = _run_blend(*args, seed=channels)
    v1, w1, ref_v1, ref_w1, c1 = _run_blend(*args, seed=channels, val_offset=1, wsum_offset=1)
    assert all(c == set() for c in c4) and all(c == {"pointer"} for c in c1), (c4, c1)
    assert torch.equal(ref_v, ref_v1) and torch.equal(ref_w, ref_w1)
    assert_bits(v4, v1, "float4 vs scalar val")
    assert_bits(w4, w1, "float4 vs scalar wsum")
    assert_bits(v4, ref_v, "val")
    assert_bits(w4, ref_w, "wsum")


# ------------------------------------------------------------------------------------------------ BlendCanvas windows
def test_blend_canvas_rejects_a_window_the_kernel_would_misread():
    g = torch.Generator().manual_seed(3)
    cv = BlendCanvas(2, 64, 96, "cuda")
    tile = torch.randn(2, 40, 64, generator=g).to(DEV)
    bad = {
        "non-square tile, no window": None,
        "[tw, th]": torch.rand(64, 40, device=DEV),
        "[th, th]": torch.rand(40, 40, device=DEV),
        "fp64": torch.rand(40, 64, device=DEV, dtype=torch.float64),
        "bf16": torch.rand(40, 64, device=DEV).bfloat16(),
        "on the CPU": torch.rand(40, 64),
        "3-d": torch.rand(1, 40, 64, device=DEV),
    }
    for what, win in bad.items():
        with pytest.raises(ValueError):
            cv.accumulate(tile, 8, 16, win)
            pytest.fail(what)
    torch.cuda.synchronize()
    assert int(torch.count_nonzero(cv.val)) == 0 and int(torch.count_nonzero(cv.wsum)) == 0     # nothing launched


@pytest.mark.parametrize("th,tw", [(40, 64), (48, 48)])
def test_blend_canvas_reads_a_strided_window_by_index(th, tw):
    """A transposed view of an asymmetric window blends exactly like its contiguous copy (and like the reference)."""
    g = torch.Generator().manual_seed(th + tw)
    win = _window(g, tw, th).t()                    # [th, tw], not contiguous, not equal to its own transpose
    assert not win.is_contiguous() and (th != tw or not torch.equal(win, win.t()))
    tiles = [(torch.randn(3, th, tw, generator=g), y0, x0) for y0, x0 in ((0, 0), (-6, 30), (50, 70))]
    ref_v, ref_w = torch.zeros(3, 80, 100), torch.zeros(80, 100)
    a, b = BlendCanvas(3, 80, 100, "cuda"), BlendCanvas(3, 80, 100, "cuda")
    win_d = win.to(DEV)
    assert not win_d.is_contiguous()
    for tile, y0, x0 in tiles:
        a.accumulate(tile.to(DEV), y0, x0, win_d)
        b.accumulate(tile.to(DEV), y0, x0, win.contiguous().to(DEV))
        _accumulate_ref(ref_v, ref_w, tile, win, y0, x0)
    assert_bits(a.val, b.val, "strided vs contiguous val")
    assert_bits(a.wsum, b.wsum, "strided vs contiguous wsum")
    assert_bits(a.val, ref_v, "val")
    assert_bits(a.wsum, ref_w, "wsum")


# ------------------------------------------------------------------------------------------------ blend_normalize
# name: (channels, h, w, out pointer offset in floats, path); the grid-stride cases hold more elements than one pass
# of the 8 x SMs x 256-thread grid covers (x 4 on the float4 path)
NORMALIZE_CASES = {
    "float4": (3, 64, 96, 0, "float4"),
    "scalar-37x41": (3, 37, 41, 0, "scalar"),
    "scalar-out-pointer+1": (3, 64, 96, 1, "scalar"),
    "float4-grid-stride": (2, 1024, 1040, 0, "float4"),
    "scalar-grid-stride": (3, 517, 519, 0, "scalar"),
}


@pytest.mark.parametrize("divisor", [1.0, 0.5, 0.3])
@pytest.mark.parametrize("case", list(NORMALIZE_CASES))
def test_blend_normalize(case, divisor):
    c, h, w, offset, path = NORMALIZE_CASES[case]
    plane, n = h * w, c * h * w
    assert (path == "float4") == (plane % 4 == 0 and offset == 0)
    if "grid-stride" in case:
        assert n > 8 * _sms() * 256 * (4 if path == "float4" else 1), (n, _sms())
    g = torch.Generator().manual_seed(n + int(divisor * 10))
    val = torch.randn(c, h, w, generator=g) * 5
    wsum = torch.rand(h, w, generator=g) * 3 + 0.01
    zero_w = torch.rand(h, w, generator=g) < 0.03          # weight sum 0: x / 0 = +-inf, and 0 / 0 = NaN where x = 0
    wsum[zero_w] = 0.0
    val[:, zero_w & (torch.rand(h, w, generator=g) < 0.5)] = 0.0
    val[torch.rand(c, h, w, generator=g) < 0.01] = -0.0    # signed zeros keep their sign
    ref = val / wsum
    if divisor != 1.0:
        ref = ref / _f32(divisor)
    assert bool(torch.isnan(ref).any()) and bool(torch.isinf(ref).any())
    v_d, w_d = val.to(DEV), wsum.to(DEV)
    out = _Buf((c, h, w), offset=offset)
    _launch(L.lib().tdx_blend_normalize, out.ptr(), v_d.data_ptr(), w_d.data_ptr(), c, plane, divisor)
    out.check(case)
    assert_bits(out.view, ref, f"{case} / {divisor}")
    assert torch.equal(v_d.cpu(), val) and torch.equal(w_d.cpu(), wsum)


# ------------------------------------------------------------------------------------------------ sched_step
def _sched_coef(which: str) -> torch.Tensor:
    """fp32 [c_skip, c_out, r, k] of a 20-step schedule: the first (first-order) step, a second-order step, and the
    last step, whose next sigma is 0 (r = 0)."""
    s = EDMDPMSolverMultistepScheduler()
    s.set_timesteps(20)
    i, second = {"first-order": (0, False), "second-order": (5, True), "r=0": (19, False)}[which]
    co = s.step_coefficients(i, second)
    coef = torch.tensor([co["c_skip"], co["c_out"], co["r"], co["k"]], dtype=F32)
    assert (float(coef[3]) != 0.0) == second and (float(coef[2]) == 0.0) == (which == "r=0")
    return coef


@pytest.mark.parametrize("which", ["first-order", "second-order", "r=0"])
@pytest.mark.parametrize("numel", [1, 7, 20480, 1_000_003], ids=lambda n: f"n{n}")
def test_sched_step(numel, which):
    if numel > 20480:
        assert numel > 8 * _sms() * 256, (numel, _sms())                   # grid-stride: more than one pass
    g = torch.Generator().manual_seed(numel + len(which))
    x = torch.randn(numel, generator=g) * 80
    f = torch.randn(numel, generator=g) * 0.6
    x0p = torch.randn(numel, generator=g) * 0.5
    coef = _sched_coef(which)
    want_x, want_x0 = _sched_update_fp32(x, f, x0p, coef)
    xs, fs, ps = _Buf((numel,), x), _Buf((numel,), f), _Buf((numel,), x0p)
    _launch(L.lib().tdx_sched_step, xs.ptr(), fs.ptr(), ps.ptr(), numel, *coef.tolist())
    for buf, what in ((xs, "sample"), (fs, "model_out"), (ps, "x0_prev")):
        buf.check(what)
    assert_bits(xs.view, want_x, "sample")
    assert_bits(ps.view, want_x0, "x0_prev")
    assert_bits(fs.view, f, "model_out (read only)")


# ------------------------------------------------------------------------------------------------ trig_mix
TRIG_AB = {"a,b>0": (math.cos(0.7), math.sin(0.7) * 0.5), "a<0": (-0.6173, 0.4119), "b<0": (0.8321, -0.2917)}


@pytest.mark.parametrize("ab", list(TRIG_AB))
@pytest.mark.parametrize("with_sample", [True, False], ids=["sample", "sample=None"])
@pytest.mark.parametrize("numel", [4, 20480, 1_200_004], ids=lambda n: f"n{n}")
def test_trig_mix(numel, with_sample, ab):
    if numel > 20480:
        assert numel > 8 * _sms() * 256 * 4, (numel, _sms())               # grid-stride: more than one pass
    a, b = (_f32(v) for v in TRIG_AB[ab])
    g = torch.Generator().manual_seed(numel + len(ab) + with_sample)
    z = torch.randn(numel, generator=g)
    z[torch.rand(numel, generator=g) < 0.05] = 0.0
    z[torch.rand(numel, generator=g) < 0.05] = -0.0
    s = torch.randn(numel, generator=g) * 2 if with_sample else torch.zeros(numel)
    want = a * s + b * z                                                   # two roundings, then one for the add
    z_d, s_d = z.to(DEV), s.to(DEV) if with_sample else None
    out = _Buf((numel,))
    _launch(L.lib().tdx_trig_mix, out.ptr(), None if s_d is None else s_d.data_ptr(), z_d.data_ptr(), numel,
            float(a), float(b))
    out.check(f"trig_mix {ab}")
    assert_bits(out.view, want, f"trig_mix {ab}")


def test_trig_mix_rejects_bad_arguments_before_any_launch():
    out, s, z = (_Buf((16,), torch.ones(16) if i else None, offset=1) for i in range(3))
    aligned = (out.g.view.data_ptr(), s.g.view.data_ptr(), z.g.view.data_ptr())
    assert all(p % 16 == 0 for p in aligned) and all(b.ptr() % 16 == 4 for b in (out, s, z))
    bad = {
        "numel 6": (aligned, 6),
        "numel 0": (aligned, 0),
        "out + 1 float": ((out.ptr(), aligned[1], aligned[2]), 8),
        "sample + 1 float": ((aligned[0], s.ptr(), aligned[2]), 8),
        "noise + 1 float": ((aligned[0], aligned[1], z.ptr()), 8),
    }
    for what, ((po, ps, pz), n) in bad.items():
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_trig_mix, DEV, po, ps, pz, n, 0.5, 0.25)
            pytest.fail(what)
    torch.cuda.synchronize()
    assert bool(torch.isnan(out.g.view[1:]).all()), "trig_mix wrote although it rejected its arguments"
    out.check("trig_mix out")


# ------------------------------------------------------------------------------------------------ pack_weighted
PACK_PLANES = {"2x2": (2, 2), "64x64": (64, 64), "1024x1028-grid-stride": (1024, 1028)}
PACK_CASES = [(n, c, p, s) for p in ("2x2", "64x64") for n in (1, 3, 16) for c in (1, 5, 6) for s in (1.0, 0.37)]
PACK_CASES += [(1, 1, "1024x1028-grid-stride", 1.0), (3, 5, "1024x1028-grid-stride", 0.37),
               (16, 1, "1024x1028-grid-stride", 0.37)]


@pytest.mark.parametrize("n_img,channels,plane,scale", PACK_CASES,
                         ids=[f"n{n}-c{c}-{p}-scale{s}" for n, c, p, s in PACK_CASES])
def test_pack_weighted(n_img, channels, plane, scale):
    h, w = PACK_PLANES[plane]
    if "grid-stride" in plane:
        assert h * w > 4 * _sms() * 256 * 4, (h * w, _sms())              # per image: more than one pass
    g = torch.Generator().manual_seed(n_img * 100 + channels * 10 + h)
    x = torch.randn(n_img, channels, h, w, generator=g) * 3
    win = _window(g, h, w)
    want = torch.cat([(x * _f32(scale)) * win, win.expand(n_img, 1, h, w)], dim=1)
    x_d, w_d = x.to(DEV), win.to(DEV)
    out = _Buf((n_img, channels + 1, h, w))
    _launch(L.lib().tdx_pack_weighted, out.ptr(), x_d.data_ptr(), w_d.data_ptr(), n_img, channels, h * w, scale)
    out.check("pack_weighted")
    assert_bits(out.view, want, "pack_weighted")


# ------------------------------------------------------------------------------------------------ window_to_cond
# (n_img, packed channels, keep, h, w, factor): keep 5 of 6 is the latent window (weight plane right after the kept
# channels), keep 4 of 6 the decoder stage's (one channel between them); 64 x 72 at factor 8 needs more than the
# 1024-block grid
COND_CASES = [(1, 6, 5, 8, 12, 1), (16, 6, 5, 8, 12, 3), (16, 6, 4, 8, 12, 3), (1, 6, 4, 5, 7, 8), (3, 2, 1, 9, 4, 3),
              (16, 6, 4, 12, 8, 8), (1, 6, 5, 64, 72, 8), (2, 6, 4, 64, 72, 8)]


@pytest.mark.parametrize("n_img,packed,keep,h,w,f", COND_CASES,
                         ids=[f"n{n}-keep{k}of{p}-{h}x{w}-f{f}" for n, p, k, h, w, f in COND_CASES])
def test_window_to_cond(n_img, packed, keep, h, w, f):
    if h * f * w * f > 1024 * 256:
        assert -(-h * f * w * f // 256) > 1024                             # grid-stride: more than one pass
    g = torch.Generator().manual_seed(n_img + packed * keep + h * w * f)
    p = torch.randn(n_img, packed, h, w, generator=g) * 4
    p[:, -1] = torch.rand(n_img, h, w, generator=g) * 2 + 0.01
    p[:, -1][torch.rand(n_img, h, w, generator=g) < 0.1] = 0.0           # weight 0: +-inf, or NaN where x = 0 too
    p[:, 0][torch.rand(n_img, h, w, generator=g) < 0.2] = 0.0
    want = (p[:, :keep] / p[:, -1:]).repeat_interleave(f, dim=2).repeat_interleave(f, dim=3)
    p_d = p.to(DEV)
    out = _Buf((n_img, keep, h * f, w * f))
    _launch(L.lib().tdx_window_to_cond, out.ptr(), p_d.data_ptr(), n_img, packed, keep, h, w, f)
    out.check("window_to_cond")
    assert_bits(out.view, want, "window_to_cond")


# ------------------------------------------------------------------------------------------------ standard_normal
def _device_standard_normal(seed: int, n: int) -> torch.Tensor:
    nbytes = int(L.lib().tdx_noise_patch_workspace_bytes(1, 1, n))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    out = _Buf((n,))
    _launch(L.lib().tdx_standard_normal, int(seed) & MASK64, n, out.ptr(), ws.data_ptr(), nbytes)
    L.call(L.lib().tdx_noise_patch_status, DEV, ws.data_ptr())             # the candidate budget covered the stream
    out.check(f"standard_normal({seed}, {n})")
    return out.view


NORMAL_GOLDEN = sorted(k for k in G.files if k.startswith("normal."))


@pytest.mark.parametrize("key", NORMAL_GOLDEN)
def test_standard_normal_matches_reference_golden(key):
    _, seed, n = key.split(".")
    got = _device_standard_normal(int(seed), int(n))
    assert_bits(got, torch.from_numpy(G[key]), key)
    assert_bits(standard_normal(int(seed), int(n)), got, f"noise.standard_normal {key}")


@pytest.mark.parametrize("seed,n", [(0, 1), (2 ** 64 - 1, 2), (77, 3), (2 ** 63 + 5, 1025), (123, 1_000_001)])
def test_standard_normal_matches_c_oracle(seed, n):
    assert_bits(_device_standard_normal(seed, n), torch.from_numpy(orng.standard_normal(seed, n)), f"{seed}.{n}")
