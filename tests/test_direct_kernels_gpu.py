"""The CUDA-core kernels around the implicit GEMM, each through its C entry point against an fp64 (or bit-exact fp32)
restatement of the contract in include/tdx.h: tdx_conv_out_run (last convolution + fused DPM-Solver++ update +
two-model guidance), tdx_embed_run (embedding and per-block modulation vectors) and tdx_attn_run (cosine attention
core).  Every output lives in a guarded buffer (tests/_igemm_ref.Guarded): a write outside the tensor fails."""
from __future__ import annotations

import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.layout import from_nc8hw8, to_nc8hw8
from terrain_diffusion_b200.models.edm_unet import _Fourier
from tests._igemm_ref import Guarded, elementwise_ratio, report

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def margins(request):
    """Worst measured error of each bound below; written to the terminal (also under -q) when the module is done."""
    found: dict = {}
    yield found
    report(request.config, [f"worst {kind}: {v:.3g}" for kind, v in sorted(found.items())])


def _guarded_like(t: torch.Tensor) -> Guarded:
    g = Guarded(tuple(t.shape), t.dtype, t.device)
    g.view.copy_(t)
    return g


def _note(margins, kind, value):
    margins[kind] = max(margins.get(kind, 0.0), value)


# ------------------------------------------------------------------------------------------------ conv_out
CONV_OUT_PAIRS = [(64, 1), (128, 1), (192, 5), (128, 6), (64, 8), (8, 3)]
CONV_OUT_SHAPES = [(1, 24, 20), (3, 5, 7), (3, 13, 9), (1, 64, 64)]


def _conv_out_weight_layout(w: torch.Tensor) -> torch.Tensor:
    """[c_out][c_in][3][3] -> the kernel's tap-major [9][c_in][1 | 8], zero padded past c_out."""
    c_out, c_in = w.shape[:2]
    wpad = 1 if c_out == 1 else 8
    w8 = torch.zeros((wpad, c_in, 3, 3), dtype=torch.float32, device=w.device)
    w8[:c_out] = w
    return w8.permute(2, 3, 1, 0).reshape(9, c_in, wpad).contiguous()


def _conv_out(x_nc8, wl, c_in, c_out, n, h, w, model_out=None, coef=None, sample=None, x0_prev=None, guide=None):
    d = L.TdxConvOutDesc()
    d.x, d.c_in, d.weight, d.c_out = x_nc8.data_ptr(), c_in, wl.data_ptr(), c_out
    d.n_img, d.height, d.width = n, h, w
    for name, buf in (("model_out", model_out), ("sched_coef", coef), ("sample", sample), ("x0_prev", x0_prev),
                      ("guide_out", guide)):
        if buf is not None:
            setattr(d, name, buf.data_ptr())
    L.check(L.lib().tdx_conv_out_run(C.byref(d), L.current_stream_ptr()))
    torch.cuda.synchronize()


def _sched_update_fp32(sample, f, x0p, coef):
    """sched_update of tdx_direct.cu in torch fp32, one rounding per operation in the kernel's order."""
    cs, co, r, k = (coef[i] for i in range(4))
    x0 = cs * sample + co * f
    t = r * sample + (1.0 - r) * x0
    return t + k * (x0 - x0p), x0


@pytest.mark.parametrize("n,h,w", CONV_OUT_SHAPES, ids=lambda v: str(v))
@pytest.mark.parametrize("c_in,c_out", CONV_OUT_PAIRS, ids=lambda v: str(v))
def test_conv_out_and_fused_update(c_in, c_out, n, h, w, margins):
    g = torch.Generator(device=DEV).manual_seed(c_in * 31 + c_out * 7 + h)
    x = torch.randn(n, c_in, h, w, generator=g, device=DEV).bfloat16().float()
    wt = torch.randn(c_out, c_in, 3, 3, generator=g, device=DEV) / (9 * c_in) ** 0.5
    x_nc8, wl = to_nc8hw8(x), _conv_out_weight_layout(wt)
    args = (x_nc8, wl, c_in, c_out, n, h, w)
    shape = (n, c_out, h, w)
    # model_out only, against the fp64 convolution; bound relative to the sum of |terms|
    mo = Guarded(shape, torch.float32, DEV)
    _conv_out(*args, model_out=mo)
    mo.check("model_out")
    f_m = mo.view.clone()
    ref = F.conv2d(x.double(), wt.double(), padding=1)
    scale = F.conv2d(x.double().abs(), wt.double().abs(), padding=1)
    err = (f_m.double() - ref).abs()
    _note(margins, "conv_out model_out (x 2^-17 sum|terms|)", float((err / (2.0 ** -17 * scale)).max()))
    assert bool((err <= 2.0 ** -17 * scale).all()), float((err / scale).max())

    # the fused DPM-Solver++ update, with a non-zero second-order term k: bit-exact against the fp32 restatement
    coef = torch.tensor([0.9173, 0.4121, 0.3377, -0.2719, 1.75], dtype=torch.float32, device=DEV)
    s0 = torch.randn(shape, generator=g, device=DEV) * 3
    p0 = torch.randn(shape, generator=g, device=DEV)
    want_s, want_x0 = _sched_update_fp32(s0, f_m, p0, coef)
    for with_model_out in (False, True):
        smp, x0p = _guarded_like(s0), _guarded_like(p0)
        mo2 = Guarded(shape, torch.float32, DEV) if with_model_out else None
        _conv_out(*args, model_out=mo2, coef=coef, sample=smp, x0_prev=x0p)
        smp.check("sample")
        x0p.check("x0_prev")
        assert torch.equal(smp.view, want_s)
        assert torch.equal(x0p.view, want_x0)
        if with_model_out:
            mo2.check("model_out")
            assert torch.equal(mo2.view, f_m)

    # two-model guidance: F = F_g + s (F_m - F_g), separately rounded, then the same update
    fg = torch.randn(shape, generator=g, device=DEV)
    f_guided = fg + coef[4] * (f_m - fg)
    want_s, want_x0 = _sched_update_fp32(s0, f_guided, p0, coef)
    smp, x0p, mo3, gd = _guarded_like(s0), _guarded_like(p0), Guarded(shape, torch.float32, DEV), _guarded_like(fg)
    _conv_out(*args, model_out=mo3, coef=coef, sample=smp, x0_prev=x0p, guide=gd)
    for buf, what in ((smp, "sample"), (x0p, "x0_prev"), (mo3, "model_out"), (gd, "guide_out")):
        buf.check(what)
    assert torch.equal(gd.view, fg)
    assert torch.equal(mo3.view, f_guided)
    assert torch.equal(smp.view, want_s)
    assert torch.equal(x0p.view, want_x0)


# ------------------------------------------------------------------------------------------------ embed
EMBED_WIDTHS = [32, 64, 96, 128, 192, 256, 384, 576, 768, 1024]
EMBED_CASES = [
    # (emb_channels, noise_dims (0 = emb_in), rows, blocks)
    (128, 64, 3, 10),
    (256, 128, 16, 20),
    (768, 192, 40, 10),
    (1024, 192, 1280, 64),
    (128, 0, 5, 10),
    (256, 0, 7, 10),
    (768, 0, 1280, 64),
    (1024, 0, 33, 30),
]


def _mp_silu64(x):
    return x * torch.sigmoid(x) / 0.596


@pytest.mark.parametrize("E,noise_dims,rows,n_blocks", EMBED_CASES,
                         ids=lambda v: str(v))
def test_embed_modulation_vectors(E, noise_dims, rows, n_blocks, margins):
    g = torch.Generator(device=DEV).manual_seed(E + noise_dims + rows)
    widths = [EMBED_WIDTHS[i % len(EMBED_WIDTHS)] for i in range(n_blocks)]
    d = L.TdxEmbedDesc()
    if noise_dims:
        labels = torch.linspace(0.003, 1.567, rows, device=DEV).flip(0).contiguous()     # a distinct label per row
        freqs = _Fourier(noise_dims, positional=True).freqs.to(DEV).contiguous()
        w_noise = (torch.randn(noise_dims, E, generator=g, device=DEV) / noise_dims ** 0.5).contiguous()
        d.noise_labels, d.noise_freqs, d.noise_weight = labels.data_ptr(), freqs.data_ptr(), w_noise.data_ptr()
        d.noise_dims = noise_dims
        y = labels.outer(freqs).double()                       # t * f rounded to fp32, as the model computes it
        pe = torch.cat([torch.sin(y), torch.cos(y)], dim=1) * 2 ** 0.5
        emb = _mp_silu64(pe @ w_noise.double())
    else:
        emb_in = torch.randn(rows, E, generator=g, device=DEV).contiguous()
        d.emb_in = emb_in.data_ptr()
        emb = emb_in.double()
    arr = (L.TdxEmbedBlock * n_blocks)()
    weights, outs = [], []
    for i, c in enumerate(widths):
        wb = (torch.randn(E, c, generator=g, device=DEV) * (0.8 / E ** 0.5)).contiguous()
        o = Guarded((rows, c), torch.float32, DEV)
        arr[i].weight, arr[i].cvec, arr[i].c_out = wb.data_ptr(), o.data_ptr(), c
        weights.append(wb)
        outs.append(o)
    d.emb_channels, d.n_img, d.n_blocks, d.blocks = E, rows, n_blocks, arr
    L.check(L.lib().tdx_embed_run(C.byref(d), L.current_stream_ptr()))
    torch.cuda.synchronize()
    for i, (wb, o) in enumerate(zip(weights, outs)):
        o.check(f"block {i} cvec")
        c = emb @ wb.double() + 1.0
        ref = c / (c.square().mean(dim=1, keepdim=True) + 1e-8).sqrt()
        err = float((o.view.double() - ref).abs().max())
        _note(margins, "embed cvec (abs)", err)
        assert err <= 2e-5, (i, widths[i], err)


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("n", [1, 5])
@pytest.mark.parametrize("tokens", [1, 40, 64, 96, 256, 262])
@pytest.mark.parametrize("heads", [1, 3, 12])
def test_attention_core(heads, tokens, n, margins):
    g = torch.Generator(device=DEV).manual_seed(heads * 1000 + tokens * 10 + n)
    C_ = heads * 64

    def draw():
        mag = 10.0 ** (4 * torch.rand(n, heads, 1, tokens, generator=g, device=DEV) - 2)    # 1e-2 .. 1e2 per token
        t = torch.randn(n, heads, 64, tokens, generator=g, device=DEV) * mag
        return t.reshape(n, C_, tokens).bfloat16().float()

    q, k, v = draw(), draw(), draw()
    dev_qkv = [to_nc8hw8(t[..., None]) for t in (q, k, v)]                  # [n][C/8][tokens][1][8]
    out = Guarded((n, C_ // 8, tokens, 1, 8), torch.bfloat16, DEV)
    d = L.TdxAttnDesc()
    d.q, d.k, d.v, d.out = dev_qkv[0].data_ptr(), dev_qkv[1].data_ptr(), dev_qkv[2].data_ptr(), out.data_ptr()
    d.n_img, d.heads, d.head_dim, d.tokens = n, heads, 64, tokens
    L.check(L.lib().tdx_attn_run(C.byref(d), L.current_stream_ptr()))
    torch.cuda.synchronize()
    out.check("attn out")
    got = from_nc8hw8(out.view)[..., 0].reshape(n, heads, 64, tokens)

    def norm(t):
        t = t.double().reshape(n, heads, 64, tokens)
        return t / (1e-4 + t.square().mean(dim=2, keepdim=True).sqrt())

    qn, kn, vn = norm(q), norm(k), norm(v)
    wts = torch.softmax(torch.einsum("nhdq,nhdk->nhqk", qn, kn) / 8.0, dim=-1)
    ref = torch.einsum("nhqk,nhdk->nhdq", wts, vn)
    ratio = elementwise_ratio(got, ref)
    _note(margins, "attention (x per-element bound)", ratio)
    assert ratio <= 1.0, ratio

