"""No C entry point reads outside, or writes into, the inputs it is given.

Every other test places its inputs in plain torch allocations, so a kernel that reads one element past an input (the
last row or column of a stencil, the tail of a vectorised loop, a halo at the plane's edge, one weight stage too many)
reads whatever the caching allocator put next to it -- usually finite data or zeros that a zero weight, a select or an
fmaxf hides.  Here every case runs three times: with plain allocations, and with every input fenced
(tests/_fence.Fenced) under pattern A and under pattern B.  It asserts that

  * every output is bit-identical across the three runs (compared as bytes, so a NaN equals a NaN),
  * every input, fences included, is byte-identical after the call, and
  * every output guard (tests/_igemm_ref.Guarded or a byte guard) is intact.

Every output compared here is deterministic run to run (the kernels' own tests assert bit-identical repeats); scratch
buffers (flow_accumulate's `state`, fill_depressions' `kind` and `flags`, the noise workspace) are only guarded.
Shapes reach the edges: sizes that are not multiples of any tile or vector width (1 x 1, 1 x w, h x 1, 33 x 37,
width 257), windows and tiles touching or overhanging each side of the plane, element counts one past a full pass of a
grid-stride kernel's capped grid, and one product-size shape per area.

tdx_program_* replay the descriptors of tdx_igemm_run / im2col / conv_out / embed / attn, which are fenced here;
tests/test_program_gpu.py checks the replay bit for bit against direct launches, so they are not repeated.
"""
from __future__ import annotations

import ctypes as C
import functools
import math
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference.relief import gaussian_taps
from terrain_diffusion_b200.layout import to_nc8hw8
from terrain_diffusion_b200.models.edm_unet import _Fourier
from tests import _igemm_ref as IR
from tests import test_igemm_plans_gpu as IP
from tests._coarse_pool_inputs import epilogue_input
from tests._coarse_view_inputs import seeded_lut
from tests._depression_inputs import fill_case, smooth_case
from tests._fence import FENCED_ARGS, Fenced, FencedStruct
from tests._igemm_surface import gpu_tests_selected, product_representatives, surface_representatives
from tests._hydrology_inputs import hydrology_case, smooth_field
from tests._minecraft_inputs import planes as mc_planes
from tests._post_inputs import field
from tests._relief_inputs import bench_field
from tests._terrain_api_inputs import planes as api_planes
from tests.test_direct_kernels_gpu import _conv_out_weight_layout

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = torch.float32
PATTERNS = (None, "A", "B")
SENTINEL8 = 0x5A
GUARD = IR.GUARD_BYTES


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _t(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)) if isinstance(a, np.ndarray) else a


_DEFAULT_ROLE = {torch.float32: "f32", torch.float64: "f64", torch.bfloat16: "bf16"}


class ByteGuarded:
    """An output of any dtype inside GUARD sentinel bytes on each side; the view starts 16-byte aligned and is filled
    with 0xFF (NaN for floats, -1 for integers) so an unwritten element shows."""

    def __init__(self, shape, dtype):
        esz = torch.empty((), dtype=dtype).element_size()
        self.nbytes = math.prod(shape) * esz
        self.raw = torch.full((2 * GUARD + -(-self.nbytes // 16) * 16,), SENTINEL8, dtype=torch.uint8, device=DEV)
        self.raw[GUARD:GUARD + self.nbytes].fill_(0xFF)
        self.view = self.raw[GUARD:GUARD + self.nbytes].view(dtype).view(shape)

    def data_ptr(self):
        return self.view.data_ptr()

    def check(self, what):
        bad = int((self.raw[:GUARD] != SENTINEL8).sum()) + int((self.raw[GUARD + self.nbytes:] != SENTINEL8).sum())
        assert bad == 0, f"{what}: {bad} bytes written outside the buffer"


class Env:
    """One run of a case: places inputs (fenced with `pattern`, or plainly for None) and guarded outputs, and records
    what the run produced."""

    def __init__(self, entry: str, pattern: str | None):
        self.entry, self.pattern = entry, pattern
        self.inputs: list = []         # (name, Fenced | FencedStruct)
        self.outputs: dict = {}        # name -> (guarded buffer, compared?)
        self.results: dict = {}        # name -> bytes produced on the host side

    def inp(self, name: str, data, role: str | None = None, host: bool = False, pitch: int | None = None,
            index_values=(-1, 0)):
        data = _t(data)
        role = role or _DEFAULT_ROLE.get(data.dtype, "int")
        f = Fenced(data, "host" if host else DEV, role, self.pattern, pitch=pitch, index_values=index_values,
                   seed=len(self.inputs))
        self.inputs.append((name, f))
        return f

    def struct(self, name: str, obj, ctype):
        """Fence a descriptor (or array of descriptors) in host memory; returns a ctypes pointer to it."""
        if self.pattern is None:
            self.inputs.append((name, None))
            return C.cast(C.pointer(obj), C.POINTER(ctype)) if not isinstance(obj, C.Array) else obj
        s = FencedStruct(obj, self.pattern)
        self.inputs.append((name, s))
        return s.pointer(ctype)

    def out(self, name: str, shape, dtype=F32, init=None, compare: bool = True):
        shape = tuple(shape)
        g = IR.Guarded(shape, dtype, DEV) if dtype in (F32, torch.bfloat16) else ByteGuarded(shape, dtype)
        if init is not None:
            g.view.copy_(_t(init).to(DEV))
        self.outputs[name] = (g, compare)
        return g

    def result(self, name: str, value):
        self.results[name] = value

    def snapshot(self) -> dict:
        got = {k: v for k, v in self.results.items()}
        for name, (g, compare) in self.outputs.items():
            if compare:
                got[name] = g.view.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes()
        return got


@dataclass
class Case:
    name: str
    entry: str
    fn: object

    def __str__(self):
        return self.name


SEEN: dict = {}            # entry point -> the argument names fenced by the cases that ran


def _as_bytes(v):
    if isinstance(v, torch.Tensor):
        return v.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes()
    return v


def run_case(case: Case):
    runs = []
    for pattern in PATTERNS:
        env = Env(case.entry, pattern)
        case.fn(env)
        torch.cuda.synchronize()
        tag = f"{case.name} [{'plain' if pattern is None else 'pattern ' + pattern}]"
        for name, f in env.inputs:
            if f is not None:
                assert f.unchanged(), f"{tag}: input {name} (or its fence) changed"
        for name, (g, _) in env.outputs.items():
            g.check(f"{tag}: {name}")
        runs.append({k: _as_bytes(v) for k, v in env.snapshot().items()})
        SEEN.setdefault(case.entry, set()).update(name for name, _ in env.inputs)
    base = runs[0]
    assert base, f"{case.name}: nothing compared"
    changed = []
    for pattern, got in zip(PATTERNS[1:], runs[1:]):
        assert got.keys() == base.keys()
        diff = [k for k in base if got[k] != base[k]]
        if diff:
            changed.append(f"pattern {pattern} changed {diff}")
    assert not changed, f"{case.name}: {'; '.join(changed)}: an input was read outside its extent"


def call(fn, *args):
    L.call(getattr(L.lib(), fn), DEV, *args)


CASES: list = []


def case(entry, *variants):
    """Register fn(env, *variant) as one case per variant, named entry[variant]."""
    def deco(fn):
        for v in variants:
            v = v if isinstance(v, tuple) else (v,)
            CASES.append(Case(f"{entry}[{','.join(str(x) for x in v)}]", entry,
                              lambda env, _fn=fn, _v=v: _fn(env, *_v)))
        return fn
    return deco


def _ptr(ctype, f):
    return C.cast(C.c_void_p(f.data_ptr()), C.POINTER(ctype))


def _rand(seed, *shape, lo=-1.0, hi=1.0):
    return (np.random.RandomState(seed).uniform(lo, hi, shape)).astype(np.float32)


# ================================================================================================= implicit GEMM
@case("tdx_igemm_choose_n", 1, 2, 3)
def _choose_n(env, n_seg):
    segs = [(128, 9), (64, 1), (64, 1)][:n_seg]
    ch = env.inp("a_channels", torch.tensor([c for c, _ in segs], dtype=torch.int32), host=True)
    tp = env.inp("a_taps", torch.tensor([t for _, t in segs], dtype=torch.int32), host=True)
    env.result("n", L.lib().tdx_igemm_choose_n(256, 2, 64, 64, _ptr(C.c_int32, ch), _ptr(C.c_int32, tp), n_seg))


@case("tdx_igemm_packed_weight_elems", 1, 2, 3)
def _packed_elems(env, n_seg):
    segs = [(128, 9), (64, 1), (192, 9)][:n_seg]
    ch = env.inp("a_channels", torch.tensor([c for c, _ in segs], dtype=torch.int32), host=True)
    tp = env.inp("a_taps", torch.tensor([t for _, t in segs], dtype=torch.int32), host=True)
    env.result("elems", L.lib().tdx_igemm_packed_weight_elems(_ptr(C.c_int32, ch), _ptr(C.c_int32, tp), n_seg, 256))


def igemm_case(c: IR.Case, env):
    acts, wts, cvec, resid = IR.make_inputs(c, DEV)

    def place(name, value):
        if name == "desc":
            return env.struct(name, value, L.TdxIgemmDesc)
        return env.inp(name, value).view

    for i, o in enumerate(IR.run_cuda(c, acts, wts, cvec, resid, place=place)):
        env.result(f"out{i}", o)


def igemm_cases() -> list:
    reps = list(product_representatives()) + list(surface_representatives()) if _gpu_run[0] else []
    return [Case(f"tdx_igemm_run[{c.name}]", "tdx_igemm_run", functools.partial(igemm_case, c))
            for c in IP.HAND_CASES + reps]


_gpu_run = [False]


# ================================================================================================= direct kernels
@case("tdx_im2col_run", (1, 1, 1, 4, 1), (2, 33, 37, 4, 1), (1, 1, 257, 4, 1), (1, 257, 1, 1, 0), (3, 64, 64, 11, 0))
def _im2col(env, n, h, w, c0, c1):
    g = torch.Generator().manual_seed(h * 1000 + w)
    d = L.TdxIm2colDesc()
    srcs = [torch.randn(n, c0, h, w, generator=g), torch.randn(n, c1, h, w, generator=g).bfloat16()]
    for i, (s, c) in enumerate(zip(srcs, (c0, c1))):
        if c:
            d.src[i] = env.inp("TdxIm2colDesc.src", s).data_ptr()
            d.src_channels[i], d.src_dtype[i] = c, int(s.dtype == torch.bfloat16)
            d.src_scale[i] = env.inp("TdxIm2colDesc.src_scale", torch.tensor([0.75 + i], dtype=F32)).data_ptr()
    ci = c0 + c1 + 1
    d.k_pad = (9 * ci + 63) // 64 * 64
    d.n_img, d.height, d.width = n, h, w
    d.out = env.out("out", (n, d.k_pad // 8, h, w, 8), torch.bfloat16).data_ptr()
    call("tdx_im2col_run", env.struct("desc", d, L.TdxIm2colDesc))


@case("tdx_conv_out_run", (1, 1, 1, 64, 1, 0), (3, 5, 7, 64, 3, 1), (2, 33, 37, 128, 8, 1), (1, 1, 257, 8, 1, 1),
      (1, 257, 1, 64, 6, 0), (1, 64, 64, 192, 5, 1))
def _conv_out(env, n, h, w, c_in, c_out, guided):
    g = torch.Generator().manual_seed(c_in * 31 + c_out + h)
    x = torch.randn(n, c_in, h, w, generator=g).bfloat16().float()
    wt = torch.randn(c_out, c_in, 3, 3, generator=g) / (9 * c_in) ** 0.5
    shape = (n, c_out, h, w)
    d = L.TdxConvOutDesc()
    d.x = env.inp("TdxConvOutDesc.x", to_nc8hw8(x)).data_ptr()
    d.weight = env.inp("TdxConvOutDesc.weight", _conv_out_weight_layout(wt)).data_ptr()
    d.c_in, d.c_out, d.n_img, d.height, d.width = c_in, c_out, n, h, w
    d.sched_coef = env.inp("TdxConvOutDesc.sched_coef", torch.tensor([0.9173, 0.4121, 0.3377, -0.2719, 1.75])
                           [:5 if guided else 4]).data_ptr()
    d.sample = env.out("sample", shape, init=torch.randn(shape, generator=g) * 3).data_ptr()
    d.x0_prev = env.out("x0_prev", shape, init=torch.randn(shape, generator=g)).data_ptr()
    d.model_out = env.out("model_out", shape).data_ptr()
    if guided:
        d.guide_out = env.inp("TdxConvOutDesc.guide_out", torch.randn(shape, generator=g)).data_ptr()
    call("tdx_conv_out_run", env.struct("desc", d, L.TdxConvOutDesc))


@case("tdx_embed_run", (128, 64, 3, 3), (256, 0, 7, 5), (768, 192, 40, 10), (1024, 0, 1, 1))
def _embed(env, E, noise_dims, rows, n_blocks):
    g = torch.Generator().manual_seed(E + noise_dims + rows)
    d = L.TdxEmbedDesc()
    if noise_dims:
        d.noise_labels = env.inp("TdxEmbedDesc.noise_labels", torch.linspace(0.003, 1.567, rows).flip(0)).data_ptr()
        d.noise_freqs = env.inp("TdxEmbedDesc.noise_freqs", _Fourier(noise_dims, positional=True).freqs).data_ptr()
        d.noise_weight = env.inp("TdxEmbedDesc.noise_weight",
                                 torch.randn(noise_dims, E, generator=g) / noise_dims ** 0.5).data_ptr()
        d.noise_dims = noise_dims
    else:
        d.emb_in = env.inp("TdxEmbedDesc.emb_in", torch.randn(rows, E, generator=g)).data_ptr()
    arr = (L.TdxEmbedBlock * n_blocks)()
    for i in range(n_blocks):
        c = (32, 64, 96, 1024, 192)[i % 5]
        arr[i].weight = env.inp("TdxEmbedBlock.weight", torch.randn(E, c, generator=g) * (0.8 / E ** 0.5)).data_ptr()
        arr[i].cvec = env.out(f"cvec{i}", (rows, c)).data_ptr()
        arr[i].c_out = c
    d.emb_channels, d.n_img, d.n_blocks = E, rows, n_blocks
    d.blocks = env.struct("TdxEmbedDesc.blocks", arr, L.TdxEmbedBlock)
    call("tdx_embed_run", env.struct("desc", d, L.TdxEmbedDesc))


@case("tdx_attn_run", (1, 1, 1), (3, 40, 2), (1, 262, 1), (12, 256, 1))
def _attn(env, heads, tokens, n):
    g = torch.Generator().manual_seed(heads * 1000 + tokens * 10 + n)
    d = L.TdxAttnDesc()
    for name in ("q", "k", "v"):
        t = (torch.randn(n, heads * 64, tokens, 1, generator=g) * 3).bfloat16().float()
        setattr(d, name, env.inp(f"TdxAttnDesc.{name}", to_nc8hw8(t)).data_ptr())
    d.out = env.out("out", (n, heads * 8, tokens, 1, 8), torch.bfloat16).data_ptr()
    d.n_img, d.heads, d.head_dim, d.tokens = n, heads, 64, tokens
    call("tdx_attn_run", env.struct("desc", d, L.TdxAttnDesc))


# ============================================================================================ blend and stage glue
def _grid_stride_elems(per_thread: int) -> int:
    """Elements one pass of a glue kernel's capped grid covers (sm * 8 blocks of 256 threads), plus one element."""
    return _sms() * 8 * 256 * per_thread + per_thread


@case("tdx_sched_step", 1, 257, "pass+1")
def _sched_step(env, n):
    n = _grid_stride_elems(1) if n == "pass+1" else n
    f = env.inp("model_out", _rand(1, n))
    s = env.out("sample", (n,), init=_t(_rand(2, n, lo=-3, hi=3)))
    x0 = env.out("x0_prev", (n,), init=_t(_rand(3, n)))
    call("tdx_sched_step", s.data_ptr(), f.data_ptr(), x0.data_ptr(), n, 0.9, 0.4, 0.3, -0.2)


# tiles overhanging every side of a 2-channel canvas, then one inside it; the float4 path and the scalar path
BLEND_LAYOUTS = {"float4": (40, 48, 16, 24, [(-8, -4), (-8, 36), (30, -12), (30, 36), (12, 12), (-16, 0)]),
                 "scalar": (33, 37, 17, 19, [(-5, -7), (-5, 25), (21, -7), (21, 25), (8, 9), (0, 0)])}


@case("tdx_blend_accumulate", "float4", "scalar")
def _blend_accumulate(env, layout):
    ch, cw, th, tw, origins = BLEND_LAYOUTS[layout]
    val = env.out("canvas_val", (2, ch, cw), init=_t(_rand(4, 2, ch, cw)))
    wsum = env.out("canvas_w", (ch, cw), init=_t(_rand(5, ch, cw, lo=0.0)))
    tile = env.inp("tile", _rand(6, 2, th, tw))
    win = env.inp("window", _rand(7, th, tw, lo=0.05))
    for y0, x0 in origins:
        call("tdx_blend_accumulate", val.data_ptr(), wsum.data_ptr(), 2, ch, cw, tile.data_ptr(), win.data_ptr(), th,
             tw, y0, x0)


@case("tdx_canvas_add", "float4", "scalar")
def _canvas_add(env, layout):
    ch, cw, th, tw, origins = BLEND_LAYOUTS[layout]
    dst = env.out("dst", (3, ch, cw), init=_t(_rand(8, 3, ch, cw)))
    tile = env.inp("tile", _rand(9, 3, th, tw))
    for y0, x0 in origins:
        call("tdx_canvas_add", dst.data_ptr(), 3, ch, cw, tile.data_ptr(), th, tw, y0, x0)


@case("tdx_blend_normalize", (1, 1), (3, 257), (2, 1028), (1, "pass+1"), (1, "pass4+1"))
def _blend_normalize(env, c, plane):
    plane = {"pass+1": _grid_stride_elems(1), "pass4+1": _grid_stride_elems(4)}.get(plane, plane)
    v = env.inp("canvas_val", _rand(10, c, plane))
    w = env.inp("canvas_w", _rand(11, plane, lo=0.1))
    o = env.out("out", (c, plane))
    call("tdx_blend_normalize", o.data_ptr(), v.data_ptr(), w.data_ptr(), c, plane, 0.5)


@case("tdx_trig_mix", 4, 260, "pass+1", "no-sample")
def _trig_mix(env, n):
    with_sample = n != "no-sample"
    n = {"pass+1": _grid_stride_elems(4), "no-sample": 1028}.get(n, n)
    s = env.inp("sample", _rand(12, n)) if with_sample else None
    z = env.inp("noise", _rand(13, n))
    o = env.out("out", (n,))
    call("tdx_trig_mix", o.data_ptr(), s.data_ptr() if s else None, z.data_ptr(), n, 0.8, 0.3)


@case("tdx_pack_weighted", (1, 1, 4), (2, 3, 260), (1, 6, "pass+1"))
def _pack_weighted(env, n, c, plane):
    plane = _sms() * 4 * 256 * 4 + 4 if plane == "pass+1" else plane
    x = env.inp("x", _rand(14, n, c, plane))
    w = env.inp("w", _rand(15, plane, lo=0.0))
    o = env.out("out", (n, c + 1, plane))
    call("tdx_pack_weighted", o.data_ptr(), x.data_ptr(), w.data_ptr(), n, c, plane, 1.7)


@case("tdx_window_to_cond", (1, 2, 1, 1, 1, 1), (2, 7, 5, 33, 37, 2), (1, 6, 5, 1, 257, 1), (1, 6, 5, 257, 1, 3),
      (1, 6, 5, 64, 64, 8))
def _window_to_cond(env, n, pc, keep, h, w, f):
    p = _rand(16, n, pc, h, w)
    p[:, -1] = np.abs(p[:, -1]) + 0.1
    packed = env.inp("packed", p)
    o = env.out("out", (n, keep, h * f, w * f))
    call("tdx_window_to_cond", o.data_ptr(), packed.data_ptr(), n, pc, keep, h, w, f)


@case("tdx_coarse_epilogue", (1, 64, 1, 0, 0), (2, 64, 2, 1, 2), (1, 64, 16, 2, 1), (3, 35, 5, 1, 2), (1, 1, 1, 0, 0),
      (16, 64, 4, 0, 0))
def _coarse_epilogue(env, n, size, pool, elev_mode, p5_mode):
    x, means, stds = epilogue_input()
    x = x[:, :size, :size].unsqueeze(0).repeat(n, 1, 1, 1).contiguous()
    s = size // pool
    o = env.out("out", (n, 7, s, s))
    call("tdx_coarse_epilogue", o.data_ptr(), env.inp("x", x).data_ptr(), env.inp("means", means).data_ptr(),
         env.inp("stds", stds).data_ptr(), env.inp("w", _rand(17, s, s, lo=0.0)).data_ptr(), n, size, pool, elev_mode,
         p5_mode, 0.5)


# ============================================================================================== elevation read-out
POST_SHAPES = [(1, 1), (1, 257), (257, 1), (33, 37), (8, 8), (512, 512)]


@case("tdx_post_normalize", *POST_SHAPES)
def _post_normalize(env, h, w):
    num = env.inp("num", field(1, h, w, 0.0, 50.0), pitch=w + 3)
    den = env.inp("den", np.abs(field(2, h, w, 1.0, 0.5)) + 0.1, pitch=w + 3)
    o = env.out("out", (h, w))
    call("tdx_post_normalize", num.data_ptr(), den.data_ptr(), w + 3, o.data_ptr(), h, w, 2.5, -1.0)


@case("tdx_post_pad_extrapolate", *POST_SHAPES)
def _pad_extrapolate(env, h, w):
    x = env.inp("x", field(3, h, w, 10.0, 20.0))
    o = env.out("out", (h + 2, w + 2))
    call("tdx_post_pad_extrapolate", x.data_ptr(), h, w, o.data_ptr())


@case("tdx_resize_aa_axis", (1, 1, 1, 1), (1, 257, 64, 1), (257, 1, 64, 0), (33, 37, 100, 1), (33, 37, 100, 0),
      (33, 37, 5, 1), (33, 37, 5, 0), (512, 512, 64, 1), (64, 512, 512, 0))
def _resize(env, h, w, out_size, axis):
    x = env.inp("x", field(4, h, w, 0.0, 30.0))
    o = env.out("out", (out_size, w) if axis == 0 else (h, out_size))
    call("tdx_resize_aa_axis", x.data_ptr(), h, w, o.data_ptr(), out_size, axis)


@case("tdx_gaussian_blur", (1, 1, 1), (2, 257, 3), (257, 2, 3), (33, 37, 31), (16, 16, 31), (512, 512, 5))
def _blur(env, h, w, k):
    x = env.inp("x", field(5, h, w, 0.0, 30.0))
    o = env.out("out", (h, w))
    call("tdx_gaussian_blur", x.data_ptr(), h, w, o.data_ptr(), k, 1.5)


@case("tdx_post_combine", *[(h, w, sq) for (h, w), sq in zip(POST_SHAPES, (0, 1, 0, 1, 1, 1))])
def _combine(env, h, w, sq):
    a = env.inp("a", field(6, h, w, 0.0, 300.0), pitch=w + 5)
    b = env.inp("b", field(7, h, w, 0.0, 30.0), pitch=w + 1)
    o = env.out("out", (h, w))
    o16 = env.out("out_i16", (h, w), torch.int16)
    call("tdx_post_combine", a.data_ptr(), w + 5, b.data_ptr(), w + 1, o.data_ptr(), o16.data_ptr(), h, w, sq)


def _edge_crops(h, w, scale, H, W, ring=0):
    """Crops touching the top-left, top-right, bottom-left and bottom-right edges of the upsampled window (with a
    `ring`-pixel margin for the Minecraft read-out's slope ring)."""
    fi, fj = h * scale - H - ring, w * scale - W - ring
    return [(ring, ring), (ring, fj), (fi, ring), (fi, fj)]


@case("tdx_terrain_upsample", (4, 5, 1, 4, 5), (3, 3, 2, 1, 1), (6, 40, 2, 9, 77), (12, 14, 8, 33, 37),
      (33, 37, 4, 100, 1), (260, 260, 4, 1024, 1024))
def _terrain_upsample(env, h, w, scale, H, W):
    p = api_planes(3, 0, 0, h, w, specials=True)
    elev = env.inp("elev", p[0])
    clim = env.inp("climate", p[1:6])
    e = env.out("elev_out", (4, H, W))
    c = env.out("climate_out", (4, 5, H, W))
    body = env.out("payload", (4, H * W * 18), torch.uint8)
    for i, (oi, oj) in enumerate(_edge_crops(h, w, scale, H, W)):
        call("tdx_terrain_upsample", elev.data_ptr(), clim.data_ptr(), h, w, scale, oi, oj, H, W, e.view[i].data_ptr(),
             c.view[i].data_ptr(), None)
        call("tdx_terrain_upsample", elev.data_ptr(), clim.data_ptr(), h, w, scale, oi, oj, H, W, None, None,
             body.view[i].data_ptr())


MC_SCAL = (50.0, 35.0, 30.0, 90.0, float(np.float32(40 * 30.0 / 90)))


@case("tdx_minecraft_readout", (5, 6, 2, 3, 5, 1), (3, 3, 2, 1, 1, 1), (12, 14, 8, 33, 37, 1), (30, 24, 4, 51, 1, 0),
      (3, 259, 1, 1, 257, 0), (35, 39, 1, 33, 37, 0), (260, 260, 4, 1024, 1024, 1))
def _minecraft(env, h, w, scale, H, W, detail):
    p = mc_planes(5, 0, 0, h, w)
    elev = env.inp("elev", p[0])
    if scale == 1:
        centre = env.inp("centre", p[0, 1:-1, 1:-1])
        clim = env.inp("climate", p[1:6, 1:-1, 1:-1])
        crops = [(1, 1)]
    else:
        centre = None
        clim = env.inp("climate", p[1:6])
        crops = _edge_crops(h, w, scale, H, W, ring=1)
    noise = env.inp("noise", _rand(18, 5, H, W))
    k = len(crops)
    outs = [env.out("elev_out", (k, H, W)), env.out("smooth_out", (k, H, W)), env.out("climate_out", (k, 5, H, W)),
            env.out("biome_out", (k, H, W), torch.int16)]
    body = env.out("payload", (k, 4 * H * W), torch.uint8)
    for i, (oi, oj) in enumerate(crops):
        args = (elev.data_ptr(), h, w, scale, oi, oj, centre.data_ptr() if centre else None, clim.data_ptr(),
                noise.data_ptr(), H, W, detail, *MC_SCAL)
        call("tdx_minecraft_readout", *args, *[o.view[i].data_ptr() for o in outs], None)
        call("tdx_minecraft_readout", *args, None, None, None, None, body.view[i].data_ptr())


# ================================================================================================ climate read-out
@case("tdx_lapse_rate", (3, 3, 3), (33, 37, 5), (3, 257, 3), (257, 3, 3), (64, 64, 7), (40, 40, 39))
def _lapse_rate(env, h, w, win):
    temp = env.inp("temp", field(8, h, w, 10.0, 8.0))
    el = env.inp("coarse_elev_sqrt", field(9, h, w, 5.0, 20.0))
    ts = env.out("t_sea", (h - win + 1, w - win + 1))
    be = env.out("beta", (h - win + 1, w - win + 1))
    call("tdx_lapse_rate", temp.data_ptr(), el.data_ptr(), h, w, win, -0.012, -0.001, -0.0065, 1e-6, 0.25,
         ts.data_ptr(), be.data_ptr())


@case("tdx_climate_sample", (12, 14, 2, 8, 33, 37), (5, 5, 2, 4, 1, 1), (7, 9, 1, 16, 1, 257), (20, 20, 4, 32, 512, 512))
def _climate_sample(env, hc, wc, crop, S, h, w):
    hs, ws = hc - 2 * crop, wc - 2 * crop
    t_sea = env.inp("t_sea", field(10, hs, ws, 15.0, 5.0))
    beta = env.inp("beta", field(11, hs, ws, -0.006, 0.001))
    coarse = env.inp("coarse", np.stack([field(12 + c, hc, wc, 0.0, 10.0) for c in range(6)]))
    elev = env.inp("elev", field(20, h, w, 200.0, 400.0))
    # windows whose pixel centres run off each side of the sampled coarse region (border-clamped), and one inside it
    span_i, span_j = hs * S, ws * S
    windows = [(-S - 3, -S - 3), (-S - 3, span_j - w + S), (span_i - h + S, -S - 3), (span_i - h + S, span_j - w + S),
               (S // 2, S // 2)]
    o = env.out("out", (len(windows), 5, h, w))
    for i, (i1, j1) in enumerate(windows):
        call("tdx_climate_sample", t_sea.data_ptr(), beta.data_ptr(), coarse.data_ptr(), 6, hc, wc, crop,
             elev.data_ptr(), i1, j1, h, w, S, 0, 0, o.view[i].data_ptr())


# =================================================================================================== relief map
def _stats_cap() -> int:
    return 4 * _sms() * 256          # elements one pass of tdx_relief_stats' grid covers


@case("tdx_relief_stats", 1, 257, "pass+1")
def _relief_stats(env, n):
    n = _stats_cap() + 1 if n == "pass+1" else n
    x = _rand(21, n, lo=-100.0, hi=900.0)
    x[::7] = np.nan
    st = env.out("stats", (3,), torch.int32)
    call("tdx_relief_stats", env.inp("elev", x).data_ptr(), n, st.data_ptr())


@case("tdx_relief_gaussian", (1, 1, (1.0,)), (1, 257, (3.0, 1.0)), (257, 1, (2.0,)), (33, 37, (20.0, 3.0)),
      (512, 512, (5.0, 1.5)))
def _relief_gaussian(env, h, w, sigmas):
    x = field(22, h, w, 100.0, 300.0)
    x[::5, ::3] = np.nan
    taps = [gaussian_taps(s) for s in sigmas]
    wts = env.inp("weights", torch.from_numpy(np.concatenate(taps).astype(np.float64)), host=True)
    rad = env.inp("radius", torch.tensor([len(t) // 2 for t in taps], dtype=torch.int32), host=True)
    n = len(sigmas)
    tmp, out = env.out("tmp", (n, h, w)), env.out("out", (n, h, w))
    call("tdx_relief_gaussian", env.inp("x", x).data_ptr(), h, w, 1, 0.0, n, _ptr(C.c_double, wts),
         _ptr(C.c_int32, rad), tmp.data_ptr(), out.data_ptr())


def _f32_bits(v) -> int:
    return int(np.float32(v).view(np.uint32))


@case("tdx_relief_shade", (2, 2, 0), (2, 257, 1), (257, 2, 0), (33, 37, 0), (33, 37, 1), (512, 512, 0))
def _relief_shade(env, h, w, user_range):
    e = bench_field(max(h, w))[:h, :w].copy()
    e[::9, ::4] = np.nan
    e[1::11] -= 400.0
    blurred = np.stack([field(23, h, w, 200.0, 300.0), field(24, h, w, 200.0, 300.0)])
    stats = np.array([int(np.isnan(e).sum()), ~_f32_bits(0.0) & 0xFFFFFFFF, _f32_bits(np.nanmax(e))], np.uint32)
    lut = np.random.RandomState(25).uniform(0, 1, (256, 3)).astype(np.float32)
    o = env.out("out", (h, w, 3))
    call("tdx_relief_shade", env.inp("elev", e).data_ptr(), env.inp("blurred", blurred).data_ptr(),
         env.inp("stats", torch.from_numpy(stats.view(np.int32))).data_ptr(), env.inp("lut", lut).data_ptr(), h, w, 1,
         0.0, 5.0, math.radians(315), math.sin(math.radians(45)), math.cos(math.radians(45)), 0.4, 0.6, user_range,
         50.0, 700.0, 0, o.data_ptr())


# ================================================================================================= explorer views
DETAIL_SIZES = [1, 3, 257, 33 * 37, "pass+1", 1024 * 1024]


def _detail_n(n):
    return _stats_cap() * 4 + 1 if n == "pass+1" else n


def _detail_plane(n):
    x = _rand(26, n, lo=-50.0, hi=3000.0)
    x[5::13] = np.nan
    return x


@case("tdx_detail_range", *DETAIL_SIZES)
def _detail_range(env, n):
    n = _detail_n(n)
    r = env.out("range", (2,), torch.int32)
    call("tdx_detail_range", env.inp("x", _detail_plane(n)).data_ptr(), n, r.data_ptr())


def _range_keys(x):
    """The tdx_detail_range keys of x's nanmin / nanmax (order-preserving, never 0)."""
    def key(v):
        b = int(np.float32(v).view(np.uint32))
        return (b ^ 0xFFFFFFFF) if b & 0x80000000 else (b | 0x80000000)
    lo, hi = np.nanmin(x), np.nanmax(x)
    return np.array([~key(lo) & 0xFFFFFFFF, key(hi)], np.uint32).view(np.int32)


@case("tdx_detail_colour", *DETAIL_SIZES)
def _detail_colour(env, n):
    n = _detail_n(n)
    x = _detail_plane(n)
    img = env.out("out", (n, 4), torch.uint8)
    call("tdx_detail_colour", env.inp("x", x).data_ptr(), n, env.inp("range", _range_keys(x)).data_ptr(),
         env.inp("lut", seeded_lut().astype(np.float32)).data_ptr(), img.data_ptr())


@case("tdx_detail_rgba8", *DETAIL_SIZES)
def _detail_rgba8(env, n):
    n = _detail_n(n)
    rgb = _rand(27, n, 3, lo=-0.2, hi=1.2)
    rgb[3::17, 1] = np.nan
    img = env.out("out", (n, 4), torch.uint8)
    call("tdx_detail_rgba8", env.inp("rgb", rgb).data_ptr(), n, img.data_ptr())


@case("tdx_detail_raw", *DETAIL_SIZES)
def _detail_raw(env, n):
    n = _detail_n(n)
    body = env.out("body", (6 * n,), torch.uint8)
    call("tdx_detail_raw", env.inp("elev", _detail_plane(n)).data_ptr(),
         env.inp("temp", _rand(28, n, lo=-20, hi=40)).data_ptr(), n, body.data_ptr())


def _coarse_sums(n):
    s = _rand(29, 7, n, lo=-3000.0, hi=3000.0)
    s[6] = np.abs(s[6]) / 1000.0
    s[6, ::11] = 0.0
    s[:, 7::19] = np.nan
    return s


COARSE_SIZES = [1, 3, 257, 33 * 37, "pass+1", 1024 * 1024]


@case("tdx_coarse_readout", *COARSE_SIZES)
def _coarse_readout(env, n):
    n = _detail_n(n)
    pl = env.out("planes", (7, n))
    r = env.out("range", (14,), torch.int32)
    call("tdx_coarse_readout", env.inp("sums", _coarse_sums(n)).data_ptr(), n, 1, pl.data_ptr(), r.data_ptr())


@case("tdx_coarse_image", *[(n, c) for n, c in zip(COARSE_SIZES, (0, 4, 2, 5, 3, 4))])
def _coarse_image(env, n, channel):
    n = _detail_n(n)
    planes = _coarse_sums(n)
    planes[6] = np.log1p(np.maximum(planes[4], 0))
    rng = np.zeros(14, np.int32)
    for p in range(7):
        rng[2 * p:2 * p + 2] = _range_keys(planes[p])
    bounds = np.array([[-500, 2000], [0, 0], [-10, 30], [0, 2000], [-1, 1e9], [5, 100]], np.float32)
    img = env.out("out", (n, 4), torch.uint8)
    call("tdx_coarse_image", env.inp("planes", planes).data_ptr(), n, channel, env.inp("range", rng).data_ptr(),
         env.inp("lut", seeded_lut().astype(np.float32)).data_ptr(), env.inp("bounds", bounds, host=True).data_ptr(),
         0xFF3, img.data_ptr())


@case("tdx_coarse_round", *COARSE_SIZES)
def _coarse_round(env, n):
    n = _detail_n(n)
    o = env.out("out", (n,))
    call("tdx_coarse_round", env.inp("x", _detail_plane(n)).data_ptr(), n, o.data_ptr())


@case("tdx_coarse_land", (1, 1, 0), (1, 257, 0), (33, 37, 3), (24, 24, 12), (257, 2, 1), (512, 512, 12))
def _coarse_land(env, h, w, half):
    ho, wo = h - 2 * half, w - 2 * half
    e = field(30, h, w, 0.0, 500.0)
    rows = env.out("rows", (h, max(wo, 0)), torch.int32) if wo > 0 else None
    mask = env.out("mask", (max(ho, 0), max(wo, 0)), torch.uint8) if ho > 0 and wo > 0 else None
    lst = env.out("list", (1 + max(ho, 0) * max(wo, 0),), torch.int32)
    call("tdx_coarse_land", env.inp("elev_m", e).data_ptr(), h, w, half, 0.5, rows.data_ptr() if rows else None,
         mask.data_ptr() if mask else None, lst.data_ptr())


# ======================================================================================================= hydrology
def _hydro_z(name):
    if name == "smooth512":
        return smooth_field(512, seed=3)
    if name == "smooth33x37":
        return smooth_field(40, seed=4)[:33, :37].copy()
    if name == "1x1":
        return np.array([[5.0]], np.float32)
    if name == "1x257":
        return field(31, 1, 257, 100.0, 80.0)
    if name == "257x1":
        return field(32, 257, 1, 100.0, 80.0)
    return hydrology_case(name)[0]


HYDRO_Z = ["1x1", "1x257", "257x1", "smooth33x37", "mixed", "edge_ocean", "neg_inf_seams", "smooth512"]
D8_OUTS = {"kmax": torch.int8, "is_sink": torch.uint8, "rr": torch.int64, "cc": torch.int64, "recv": torch.int32,
           "indeg": torch.int32}


def _d8_plain(z):
    """rr, cc, is_sink, recv, indeg of tdx_flow_d8 in plain allocations: the inputs of the later steps."""
    h, w = z.shape
    zd = _t(z).to(DEV)
    o = {k: torch.empty((h, w), dtype=dt, device=DEV) for k, dt in D8_OUTS.items()}
    flags = torch.zeros(1, dtype=torch.int32, device=DEV)
    call("tdx_flow_d8", zd.data_ptr(), h, w, 1e-3, *[o[k].data_ptr() for k in D8_OUTS], flags.data_ptr())
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


@case("tdx_flow_d8", *HYDRO_Z)
def _flow_d8(env, name):
    z = _hydro_z(name)
    h, w = z.shape
    outs = [env.out(k, (h, w), dt) for k, dt in D8_OUTS.items()]
    flags = env.out("flags", (1,), torch.int32)
    call("tdx_flow_d8", env.inp("z", z).data_ptr(), h, w, 1e-3, *[o.data_ptr() for o in outs], flags.data_ptr())


@case("tdx_flow_link", *HYDRO_Z)
def _flow_link(env, name):
    z = _hydro_z(name)
    h, w = z.shape
    d8 = _d8_plain(z)
    recv, indeg = env.out("recv", (h, w), torch.int32), env.out("indeg", (h, w), torch.int32)
    flags = env.out("flags", (1,), torch.int32)
    call("tdx_flow_link", env.inp("z", z).data_ptr(), env.inp("rr", d8["rr"], "index", index_values=(0, h - 1)).data_ptr(),
         env.inp("cc", d8["cc"], "index", index_values=(0, w - 1)).data_ptr(),
         env.inp("is_sink", d8["is_sink"], "int").data_ptr(), h, w, recv.data_ptr(), indeg.data_ptr(), flags.data_ptr())


@case("tdx_flow_accumulate", *HYDRO_Z)
def _flow_accumulate(env, name):
    z = _hydro_z(name)
    n = z.size
    d8 = _d8_plain(z)
    state = env.out("state", (n,), torch.int64, compare=False)
    a = env.out("A", (n,))
    call("tdx_flow_accumulate", env.inp("z", z).data_ptr(), n, env.inp("recv", d8["recv"], "index").data_ptr(),
         env.inp("indeg", d8["indeg"], "int").data_ptr(), state.data_ptr(), a.data_ptr())


@case("tdx_flow_indicator", (1, 1, 1), (1, 257, 1), (257, 1, 1), (33, 37, 3), (33, 37, 8), (32, 40, 8), (24, 24, 4),
      (512, 512, 8))
def _flow_indicator(env, h, w, k):
    a = np.floor(_rand(33, h, w, lo=0.0, hi=1000.0))
    a[::6, ::5] = 0.0
    oh, ow = (h // k, w // k) if k > 1 else (h, w)
    o = env.out("out", (oh, ow))
    call("tdx_flow_indicator", env.inp("A", a).data_ptr(), h, w, k, o.data_ptr())


@case("tdx_fill_depressions", "pits8", "pits4", "nodata", "inf_land", "row", "col", "two", "big", "1x1", "1x257")
def _fill(env, name):
    if name in ("1x1", "1x257"):
        z, kw = _hydro_z(name), {}
    else:
        z, kw = fill_case(name)
    h, w = z.shape
    out = env.out("out", (h, w))
    kind = env.out("kind", (h, w), torch.uint8, compare=False)
    flags = env.out("flags", (32,), torch.int32, compare=False)
    passes = C.c_int32(-1)
    call("tdx_fill_depressions", env.inp("height", z).data_ptr(), h, w, float(np.float32(kw.get("epsilon", 1e-3))),
         kw.get("connectivity", 8), float(kw.get("nodata", float("nan"))), out.data_ptr(), kind.data_ptr(),
         flags.data_ptr(), C.byref(passes))
    env.result("passes", passes.value)


@case("tdx_smooth_river_bumps", "nan", "iter1", "params", "steep", "two", "plateau", "2x257", "257x2", "512")
def _smooth(env, name):
    if name in ("2x257", "257x2", "512"):
        z = {"2x257": field(34, 2, 257, 300.0, 200.0), "257x2": field(35, 257, 2, 300.0, 200.0),
             "512": smooth_field(512, seed=5)}[name]
        kw = {}
    else:
        z, kw = smooth_case(name)
    h, w = z.shape
    out = env.out("out", (h, w))
    sc = env.out("scratch", (h, w), compare=False)
    call("tdx_smooth_river_bumps", env.inp("height", z).data_ptr(), h, w, float(np.float32(kw.get("slope_thresh", 50.0))),
         float(np.float32(kw.get("smooth_strength", 0.3))), kw.get("iterations", 3), out.data_ptr(), sc.data_ptr())


# ============================================================================================ noise and synthesis
@case("tdx_noise_patches", (1, 1, 1, 1, 16, 16), (3, 33, 37, 2, 16, 16), (2, 1, 257, 1, 64, 64), (4, 64, 64, 5, 64, 64))
def _noise_patches(env, n, h, w, c, th, tw):
    ys = env.inp("y0s", torch.tensor([-37 + 50 * i for i in range(n)], dtype=torch.int64), "index", host=True)
    xs = env.inp("x0s", torch.tensor([91 - 29 * i for i in range(n)], dtype=torch.int64), "index", host=True)
    nb = L.lib().tdx_noise_patches_workspace_bytes(c, th, tw)
    ws = env.out("workspace", (nb,), torch.uint8, compare=False)
    ws.view.zero_()
    o = env.out("out", (n, c, h, w))
    call("tdx_noise_patches", 12345, n, _ptr(C.c_int64, ys), _ptr(C.c_int64, xs), h, w, c, th, tw, o.data_ptr(),
         ws.data_ptr(), nb)


@case("tdx_fbm_perlin", (1, 1, 1), (3, 1, 257), (2, 257, 1), (8, 33, 37), (5, 512, 512))
def _fbm(env, n, h, w):
    seeds = env.inp("seeds", torch.arange(n, dtype=torch.int32) * 7 + 3, host=True)
    freq = env.inp("frequency", torch.linspace(0.01, 0.05, n), host=True)
    octv = env.inp("octaves", torch.tensor([(1, 4, 2, 16, 4, 3, 8, 5)[k] for k in range(n)], dtype=torch.int32),
                   host=True)
    lac = env.inp("lacunarity", torch.full((n,), 2.0), host=True)
    gain = env.inp("gain", torch.full((n,), 0.5), host=True)
    o = env.out("out", (n, h, w))
    call("tdx_fbm_perlin", n, seeds.data_ptr(), freq.data_ptr(), octv.data_ptr(), lac.data_ptr(), gain.data_ptr(),
         -17, 4093, h, w, o.data_ptr())


def _tables(n_knots=64):
    t = np.empty((5, 2, n_knots), np.float64)
    for f in range(5):
        t[f, 0] = np.linspace(-0.9, 0.9, n_knots) ** 3
        t[f, 1] = np.cumsum(np.random.RandomState(40 + f).uniform(0.5, 2.0, n_knots)) * (f + 1)
    return t


SYN_FIN, SYN_SQRT, SYN_IMP, SYN_RAW = 1, 2, 4, 8


@case("tdx_synthetic_map", ("noise", 1, 1), ("noise", 33, 37), ("finalize", 1, 257), ("import", 33, 37),
      ("input", 257, 1), ("raw", 33, 37), ("import", 512, 512))
def _synthetic(env, kind, h, w):
    mode = {"noise": 0, "finalize": SYN_FIN | SYN_SQRT, "import": SYN_IMP | SYN_FIN, "input": SYN_SQRT,
            "raw": SYN_RAW | SYN_IMP | SYN_FIN}[kind]
    raw = kind == "raw"
    tables = None if raw else env.inp("tables", _tables())
    seeds = freq = None
    inp = None
    if kind in ("input", "raw"):
        inp = env.inp("input", _rand(41, 5, h, w, lo=-0.8, hi=0.8) * (1000.0 if raw else 1.0))
    else:
        seeds = env.inp("seeds", torch.tensor([11, 22, 33, 44, 55], dtype=torch.int32), host=True)
        freq = env.inp("frequency", torch.tensor([1.5, 3, 3, 3, 3], dtype=F32) / 256, host=True)
    scalars = env.inp("scalars", torch.tensor([0.3, 1.2, 2.0, 9.0, 7.0], dtype=F32), host=True) \
        if mode & SYN_FIN else None
    imp = [None, None, None, 0]
    if mode & SYN_IMP:
        # rasters 0 and 3 cover parts of the window (one spans its top-left corner, one its bottom-right); channel 2
        # falls back to its default outside everything
        r0 = env.inp("imp_values[0]", _rand(42, h // 2 + 1, w // 2 + 1, lo=-100, hi=100))
        r3 = env.inp("imp_values[3]", _rand(43, h, w, lo=0, hi=50))
        ptrs = torch.tensor([r0.data_ptr(), 0, 0, r3.data_ptr(), 0], dtype=torch.int64)
        vals = env.inp("imp_values", ptrs, "index", host=True, index_values=(0, 0))
        boxes = env.inp("imp_boxes", torch.tensor([[-5, 7, h // 2 + 1, w // 2 + 1], [0, 0, 0, 0], [0, 0, 0, 0],
                                                   [-5 + h // 2, 7 + w // 2, h, w], [0, 0, 0, 0]], dtype=torch.int64),
                        host=True)
        dflt = env.inp("imp_defaults", torch.tensor([0, 0, 4.5, 0, 0], dtype=F32), host=True)
        imp = [vals.data_ptr(), boxes.data_ptr(), dflt.data_ptr(), 0b00100]
    o = env.out("out", (5, h, w))
    call("tdx_synthetic_map", tables.data_ptr() if tables else None, 64, seeds.data_ptr() if seeds else None,
         freq.data_ptr() if freq else None, scalars.data_ptr() if scalars else None, -5, 7, h, w,
         inp.data_ptr() if inp else None, mode, *imp, o.data_ptr())


# ========================================================================================================= tests
def pytest_generate_tests(metafunc):
    if metafunc.function.__name__ == "test_inputs_are_read_inside_their_extent":
        _gpu_run[0] = gpu_tests_selected(metafunc.config)
        cases = CASES + igemm_cases()
        metafunc.parametrize("c", cases, ids=[c.name for c in cases])


def test_inputs_are_read_inside_their_extent(c):
    run_case(c)


def test_every_declared_argument_is_fenced():
    """Every argument tests/_fence.FENCED_ARGS claims is fenced by at least one case that ran (skipped when only some
    cases ran), and every entry point there has a case."""
    entries = {c.entry for c in CASES} | {"tdx_igemm_run"}
    assert entries == set(FENCED_ARGS), sorted(entries ^ set(FENCED_ARGS))
    if set(SEEN) != entries:
        pytest.skip("only some cases ran")
    missing = {e: sorted(set(FENCED_ARGS[e]) - SEEN[e]) for e in FENCED_ARGS if set(FENCED_ARGS[e]) - SEEN[e]}
    assert not missing, missing
    extra = {e: sorted({n.split("[")[0] for n in SEEN[e]} - set(FENCED_ARGS[e])) for e in SEEN}
    extra = {e: v for e, v in extra.items() if v}
    assert not extra, f"fenced but not declared in FENCED_ARGS: {extra}"
