"""NaN and +-inf through every U-Net entry point, against fp64 references that keep them (tests/_nonfinite.py).

Each kernel gets chosen elements poisoned -- interior, image corners and borders (where zero padding applies), both
sides of the 16 x 8 M-tile seams, the first and the last image of a batch -- and must put NaN, +inf and -inf in
exactly the reference's positions, every finite element within the bound its existing test uses, and every image
that was not poisoned bit for bit where a clean run puts it: a tile, cluster or workspace that crossed images would
carry the poison over.  The whole decoder, coarse and base forwards and the coarse stage follow, with one NaN
conditioning pixel (the reference feeds imported rasters and a user conditioning_fn into the coarse solve unfiltered).
Outputs live in guarded buffers (tests/_igemm_ref.Guarded).
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import WorldPipeline
from terrain_diffusion_b200.inference.stages import coarse_stage_tile, coarse_stage_tiles
from terrain_diffusion_b200.inference.tiling import linear_weight_window
from terrain_diffusion_b200.layout import from_nc8hw8, to_nc8hw8
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.models.edm_unet import _Fourier
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests import _igemm_ref as IR
from tests import _igemm_surface as S
from tests import _nonfinite as NF
from tests._stage_inputs import SEED, stage_inputs
from tests._capture import CONFIGS
from tests.test_direct_kernels_gpu import _conv_out, _conv_out_weight_layout, _guarded_like, _sched_update_fp32

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
NAN, INF = float("nan"), float("inf")


def _seam_pixels(h, w):
    """(y, x, value) poison of one image: the corner, both sides of the first 16 x 8 tile seam, the interior, the far
    border and corner."""
    px = [(0, 0, NAN), (h // 2, w // 2 + 1, NAN), (h - 1, w // 2, NAN)]
    if h > 16:
        px += [(15, min(w - 1, 3), NAN), (16, min(w - 1, 3), NAN)]
    if w > 8:
        px += [(min(h - 1, 5), 7, NAN), (min(h - 1, 9), 8, NAN)]
    return px


def _inf_pixels(h, w):
    return [(h - 1, w - 1, INF), (0, w // 2, -INF), (h // 2, 0, INF)]


def _poison_images(n):
    """First and last image poisoned (NaN in the first, +-inf in the last); the ones between stay clean."""
    return [0] if n == 1 else [0, n - 1]


def _poison_plane(t, img, pixels, channel):
    for y, x, v in pixels:
        t[img, channel, y, x] = v


# ------------------------------------------------------------------------------------------------ tdx_igemm_run
def _clip_cases():
    """The hand-written clip cases of tests/_igemm_ref.py, and each with the clip off."""
    out = []
    for c in IR.default_cases():
        if c.clip > 0:
            out += [c, dataclasses.replace(c, name=c.name + "_off", clip=0.0)]
    return out


WHERE = ("a", "resid", "cvec", "resid_inv")


def _applies(case, where):
    if where == "resid":
        return bool(case.epi & L.EPI_RESID)
    if where == "cvec":
        return bool(case.epi & L.EPI_EMB_SILU)
    if where == "resid_inv":
        return bool(case.epi & L.EPI_RESID) and case.resid_inv
    return True


def pytest_generate_tests(metafunc):
    if metafunc.function.__name__ == "test_igemm_keeps_nan_and_inf":
        reps = list(S.group_representatives()) + _clip_cases() if S.gpu_tests_selected(metafunc.config) else ()
        metafunc.parametrize("case", reps, ids=lambda c: c.name)


@pytest.mark.parametrize("where", WHERE)
def test_igemm_keeps_nan_and_inf(case, where):
    """One launch per epilogue signature and plan variant of the surface (and the clip cases): NaN and +-inf in the A
    operands, the residual, the modulation vector or the residual's pixel-norm plane, in turn."""
    if not _applies(case, where):
        pytest.skip(f"the launch reads no {where}")
    acts, wts, cvec, resid = IR.make_inputs(case, DEV)
    clean = IR.run_cuda(case, acts, wts, cvec, resid)
    imgs = _poison_images(case.n)
    acts, cvec, resid = [a.clone() for a in acts], cvec.clone(), resid.clone()
    resid_inv = None
    if where == "a":
        for s, a in enumerate(acts):          # every segment: the first NaN, the last +-inf, at different pixels
            ch = (3 * s + 1) % a.shape[1]
            _poison_plane(a, imgs[0], _seam_pixels(case.h, case.w)[s::len(acts)] or [(0, 0, NAN)], ch)
            if len(imgs) > 1:
                _poison_plane(a, imgs[-1], _inf_pixels(case.h, case.w)[s % 3:s % 3 + 1], ch)
    elif where == "resid":
        rh, rw = resid.shape[2:]
        _poison_plane(resid, imgs[0], _seam_pixels(rh, rw), 5)
        if len(imgs) > 1:
            _poison_plane(resid, imgs[-1], _inf_pixels(rh, rw), 9 % case.cout)
    elif where == "cvec":
        cvec[imgs[0], 5] = NAN                # inf * a value near 0 would take fp32's sign: NaN only
        cvec[imgs[-1], case.cout - 1] = NAN
    else:
        resid_inv = (1.0 / (1e-4 + resid.double().square().mean(dim=1).sqrt())).float().contiguous()
        rh, rw = resid.shape[2:]
        for y, x, v in _seam_pixels(rh, rw):
            resid_inv[imgs[0], y, x] = v
        resid_inv[imgs[-1], rh - 1, 0] = NAN
    got = IR.run_cuda(case, acts, wts, cvec, resid, resid_inv=resid_inv)
    sel = imgs
    refs = NF.igemm_reference(case, [a[sel] for a in acts], wts, cvec[sel], resid[sel],
                              None if resid_inv is None else resid_inv[sel], device=DEV)
    saw_nonfinite = False
    for i, (g, c, r) in enumerate(zip(got, clean, refs)):
        what = f"{case.name} {where} {'rms_out' if i == len(case.outs) else f'out{i}'}"
        NF.assert_matches(g[sel], r, what)
        saw_nonfinite |= not bool(torch.isfinite(r).all())
        rest = [j for j in range(case.n) if j not in imgs]
        assert torch.equal(g[rest], c[rest]), f"{what}: an image that was not poisoned changed"
    assert saw_nonfinite, f"{case.name} {where}: the poison reached no output"


# ------------------------------------------------------------------------------------------------ tdx_im2col_run
def _im2col(srcs, scales, n, h, w):
    """One tdx_im2col_run of (fp32 [n, 1, h, w], bf16 [n, 4, h, w]) sources; returns [n, 64, h, w] fp32 from bf16."""
    d = L.TdxIm2colDesc()
    for i, (s, sc) in enumerate(zip(srcs, scales)):
        d.src[i] = s.data_ptr()
        d.src_channels[i] = s.shape[1]
        d.src_dtype[i] = 0 if s.dtype == torch.float32 else 1
        d.src_scale[i] = sc.data_ptr() if sc is not None else None
    out = IR.Guarded((n, 8, h, w, 8), torch.bfloat16, DEV)
    d.out, d.k_pad, d.n_img, d.height, d.width = out.data_ptr(), 64, n, h, w
    L.check(L.lib().tdx_im2col_run(C.byref(d), L.current_stream_ptr()))
    torch.cuda.synchronize()
    out.check("im2col out")
    return from_nc8hw8(out.view)


def _im2col_ref(srcs, scales, n, h, w):
    """k = tap * 6 + c: source channel c (scaled, rounded to bf16) at the tap's neighbour, 1.0 for c == 5 inside the
    image, exact zeros for padded taps and for k >= 54."""
    x = torch.cat([s.float() * (sc if sc is not None else 1.0) for s, sc in zip(srcs, scales)], dim=1).cpu()
    x = torch.cat([x, torch.ones(n, 1, h, w)], dim=1)
    xp = F.pad(x, (1, 1, 1, 1))
    out = torch.zeros(n, 64, h, w)
    for tap in range(9):
        dy, dx = tap // 3, tap % 3
        out[:, tap * 6:tap * 6 + 6] = xp[:, :, dy:dy + h, dx:dx + w]
    return out.bfloat16().float()


@pytest.mark.parametrize("poison", ["fp32", "bf16", "scale"])
def test_im2col_keeps_nan_and_inf_and_pads_with_exact_zeros(poison):
    n, h, w = 3, 20, 24
    g = torch.Generator(device=DEV).manual_seed(3)
    s0 = torch.randn(n, 1, h, w, generator=g, device=DEV)
    s1 = torch.randn(n, 4, h, w, generator=g, device=DEV).bfloat16()
    sc = [torch.tensor([0.7], device=DEV), torch.tensor([1.3], device=DEV)]
    clean = _im2col([s0, s1], sc, n, h, w)
    if poison == "fp32":
        _poison_plane(s0, 0, _seam_pixels(h, w), 0)
        _poison_plane(s0, n - 1, _inf_pixels(h, w), 0)
    elif poison == "bf16":
        _poison_plane(s1, 0, _seam_pixels(h, w), 2)
        _poison_plane(s1, n - 1, _inf_pixels(h, w), 3)
    else:
        sc[1] = torch.tensor([NAN], device=DEV)
    got = _im2col([s0, s1], sc, n, h, w)
    want = _im2col_ref([s0, s1], sc, n, h, w)
    NF.assert_same_bits(got, want, f"im2col {poison}")
    assert bool(torch.isnan(got).any())
    zeros = want == 0
    assert bool((got[zeros] == 0).all()) and not bool(torch.signbit(got[:, 54:]).any())
    if poison != "scale":
        assert torch.equal(got[1], clean[1])


# ------------------------------------------------------------------------------------------------ tdx_conv_out_run
@pytest.mark.parametrize("c_in,c_out", [(64, 1), (128, 6)])
@pytest.mark.parametrize("poison", ["x", "sample", "x0_prev", "guide_out"])
@pytest.mark.parametrize("fused", ["model_out", "update", "guided"])
def test_conv_out_keeps_nan_and_inf(c_in, c_out, poison, fused):
    if poison in ("sample", "x0_prev") and fused == "model_out" or poison == "guide_out" and fused != "guided":
        pytest.skip("the launch reads no such input")
    n, h, w = 3, 24, 20
    g = torch.Generator(device=DEV).manual_seed(c_in + c_out)
    x = torch.randn(n, c_in, h, w, generator=g, device=DEV).bfloat16().float()
    wt = torch.randn(c_out, c_in, 3, 3, generator=g, device=DEV) / (9 * c_in) ** 0.5
    shape = (n, c_out, h, w)
    s0 = torch.randn(shape, generator=g, device=DEV) * 3
    p0 = torch.randn(shape, generator=g, device=DEV)
    fg = torch.randn(shape, generator=g, device=DEV)
    coef = torch.tensor([0.9173, 0.4121, 0.3377, -0.2719, 1.75], device=DEV)
    target = {"x": x, "sample": s0, "x0_prev": p0, "guide_out": fg}[poison]
    _poison_plane(target, 0, _seam_pixels(h, w), 0 if poison != "x" else 9)
    _poison_plane(target, n - 1, _inf_pixels(h, w), c_out - 1 if poison != "x" else 17)
    wl = _conv_out_weight_layout(wt)
    args = (to_nc8hw8(x), wl, c_in, c_out, n, h, w)
    mo = IR.Guarded(shape, torch.float32, DEV)
    _conv_out(*args, model_out=mo)
    mo.check("model_out")
    f_m = mo.view.clone()
    ref = F.conv2d(x.double().cpu(), wt.double().cpu(), padding=1)
    finite = NF.assert_same_nonfinite(f_m, ref, "conv_out model_out")
    scale = F.conv2d(x.double().cpu().nan_to_num(0, 0, 0).abs(), wt.double().cpu().abs(), padding=1)
    assert bool(((f_m.double().cpu() - ref).abs() <= 2.0 ** -17 * scale)[finite].all())
    if fused == "model_out":
        return
    smp, x0p = _guarded_like(s0), _guarded_like(p0)
    mo2 = IR.Guarded(shape, torch.float32, DEV)
    f = f_m
    gd = None
    if fused == "guided":
        gd = _guarded_like(fg)
        f = fg + coef[4] * (f_m - fg)
    _conv_out(*args, model_out=mo2, coef=coef, sample=smp, x0_prev=x0p, guide=gd)
    for buf, what in ((smp, "sample"), (x0p, "x0_prev"), (mo2, "model_out")):
        buf.check(what)
    want_s, want_x0 = _sched_update_fp32(s0, f, p0, coef)
    NF.assert_same_bits(mo2.view, f, f"conv_out {fused} model_out")
    NF.assert_same_bits(smp.view, want_s, f"conv_out {fused} sample")
    NF.assert_same_bits(x0p.view, want_x0, f"conv_out {fused} x0_prev")
    assert not bool(torch.isfinite(smp.view).all())
    assert bool(torch.isfinite(smp.view[1]).all())


# ------------------------------------------------------------------------------------------------ tdx_attn_run
def _attn(q, k, v, heads):
    n, c, tokens = q.shape
    dev_qkv = [to_nc8hw8(t[..., None]) for t in (q, k, v)]
    out = IR.Guarded((n, c // 8, tokens, 1, 8), torch.bfloat16, DEV)
    d = L.TdxAttnDesc()
    d.q, d.k, d.v, d.out = dev_qkv[0].data_ptr(), dev_qkv[1].data_ptr(), dev_qkv[2].data_ptr(), out.data_ptr()
    d.n_img, d.heads, d.head_dim, d.tokens = n, heads, 64, tokens
    L.check(L.lib().tdx_attn_run(C.byref(d), L.current_stream_ptr()))
    torch.cuda.synchronize()
    out.check("attn out")
    return from_nc8hw8(out.view)[..., 0]


@pytest.mark.parametrize("value", [NAN, INF, -INF], ids=["nan", "+inf", "-inf"])
@pytest.mark.parametrize("which", ["q", "k", "v"])
@pytest.mark.parametrize("tokens", [64, 262])
def test_attention_keeps_nan_and_turns_inf_into_nan(which, value, tokens):
    n, heads = 3, 3
    g = torch.Generator(device=DEV).manual_seed(tokens)
    q, k, v = (torch.randn(n, heads * 64, tokens, generator=g, device=DEV).bfloat16().float() for _ in range(3))
    clean = _attn(q, k, v, heads)
    t = {"q": q, "k": k, "v": v}[which]
    tok = tokens - 1
    t[1, 64 + 11, tok] = value                   # image 1, head 1, one channel of the last token
    got = _attn(q, k, v, heads)
    ref = NF.attention_reference(q, k, v, heads)
    NF.assert_matches(got, ref, f"attention {which}")
    nan = torch.isnan(got.reshape(n, heads, 64, tokens))
    # +-inf goes through x / (eps + rms) as NaN in its own channel and 0 in the others, as the reference's does
    if which == "q":                              # a poisoned query: its own row
        assert bool(nan[1, 1, :, tok].all()) and int(nan.sum()) == 64
    elif which == "k" or value != value:          # a poisoned key, or a NaN value: every query of the head
        assert bool(nan[1, 1].all()) and int(nan.sum()) == 64 * tokens
    else:                                         # an infinite value: its channel of every query
        assert bool(nan[1, 1, 11].all()) and int(nan.sum()) == tokens
    other = torch.ones(n, heads, dtype=torch.bool)
    other[1, 1] = False
    a, b = got.reshape(n, heads, 64, tokens), clean.reshape(n, heads, 64, tokens)
    assert torch.equal(a[other], b[other])


# ------------------------------------------------------------------------------------------------ tdx_embed_run
@pytest.mark.parametrize("path", ["noise_labels", "emb_in"])
def test_embed_nan_row_poisons_only_its_modulation_vectors(path):
    E, rows, widths = 256, 5, [64, 128, 192, 768]
    g = torch.Generator(device=DEV).manual_seed(9)
    noise_dims = 128

    def run(poison):
        d = L.TdxEmbedDesc()
        keep = []
        if path == "noise_labels":
            labels = torch.linspace(0.003, 1.567, rows, device=DEV).contiguous()
            if poison:
                labels[2] = NAN
            freqs = _Fourier(noise_dims, positional=True).freqs.to(DEV).contiguous()
            wn = (torch.randn(noise_dims, E, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
                  / noise_dims ** 0.5).contiguous()
            d.noise_labels, d.noise_freqs, d.noise_weight, d.noise_dims = (labels.data_ptr(), freqs.data_ptr(),
                                                                           wn.data_ptr(), noise_dims)
            keep += [labels, freqs, wn]
        else:
            emb_in = torch.randn(rows, E, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
            if poison:
                emb_in[2, 17] = NAN
            d.emb_in = emb_in.data_ptr()
            keep.append(emb_in)
        arr = (L.TdxEmbedBlock * len(widths))()
        outs = []
        for i, c in enumerate(widths):
            wb = (torch.randn(E, c, generator=torch.Generator(device=DEV).manual_seed(10 + i), device=DEV)
                  * (0.8 / E ** 0.5)).contiguous()
            o = IR.Guarded((rows, c), torch.float32, DEV)
            arr[i].weight, arr[i].cvec, arr[i].c_out = wb.data_ptr(), o.data_ptr(), c
            keep.append(wb)
            outs.append(o)
        d.emb_channels, d.n_img, d.n_blocks, d.blocks = E, rows, len(widths), arr
        L.check(L.lib().tdx_embed_run(C.byref(d), L.current_stream_ptr()))
        torch.cuda.synchronize()
        for i, o in enumerate(outs):
            o.check(f"block {i} cvec")
        return [o.view.clone() for o in outs]

    clean, got = run(False), run(True)
    for c, o in zip(clean, got):
        assert bool(torch.isnan(o[2]).all())
        rest = [0, 1, 3, 4]
        assert torch.equal(o[rest], c[rest])


# ------------------------------------------------------------------------------------------------ whole forwards
FORWARDS = {"decoder": (3, 64, 2), "coarse": (3, 64, 8), "base": (3, 64, 3)}   # n, side, poisoned input channel


def _oracle_inputs(cfg, x, t, cond):
    sd = {k: v.double() if v.is_floating_point() else v
          for k, v in ounet.procedural_state_dict(cfg, seed=0).items()}
    return sd, x.double().cpu(), t.double().cpu(), [c.double().cpu() for c in cond]


@pytest.mark.parametrize("name", list(FORWARDS))
def test_forward_with_one_nan_conditioning_pixel(name):
    cfg = CONFIGS[name]
    n, hw, ch = FORWARDS[name]
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
    m = m.to(DEV)
    g = torch.Generator().manual_seed(21)
    x = torch.randn(n, cfg["in_channels"], hw, hw, generator=g)
    t = torch.atan(torch.exp(torch.randn(n, generator=g) * 1.5) / 0.5)
    cond = [(torch.randn(n, dim, generator=g) if kind == "tensor" else torch.randn(n, generator=g))
            for kind, dim, _ in cfg.get("conditional_inputs") or []]
    dcond = [c.to(DEV) for c in cond]
    clean = m(x.to(DEV), t.to(DEV), dcond).clone()
    xp = x.clone()
    xp[1, ch, 37, 22] = NAN                        # image 1 of 3: one conditioning pixel
    first = m(xp.to(DEV), t.to(DEV), dcond).clone()     # the planned program (captured on its first run)
    replay = m(xp.to(DEV), t.to(DEV), dcond).clone()    # and its graph replay
    assert torch.equal(torch.isnan(first), torch.isnan(replay))
    keep = ~torch.isnan(first)
    assert torch.equal(first[keep], replay[keep]), "graph replay differs"
    assert torch.equal(first[[0, 2]], clean[[0, 2]]), "the NaN reached another image"
    sd, x64, t64, c64 = _oracle_inputs(cfg, xp[1:2], t[1:2], [c[1:2] for c in cond])
    with torch.no_grad():
        ref = ounet.unet_forward(sd, cfg, x64, t64, c64)
    finite = NF.assert_same_nonfinite(first[1:2], ref, f"{name} forward")
    assert not bool(finite.all()), f"{name}: the NaN reached no output"
    assert NF.finite_rel_rms(first[1:2], ref, finite) <= 1.0e-2


# ------------------------------------------------------------------------------------------------ the coarse stage
@pytest.fixture(scope="module")
def coarse_model():
    m = EDMUnet2D(**CONFIGS["coarse"]).eval()
    m.load_state_dict(ounet.procedural_state_dict(CONFIGS["coarse"], seed=0))
    return m.to(DEV)


def test_coarse_stage_with_nan_conditioning_cells(coarse_model):
    """A conditioning_fn that returns NaN cells in one window: that window's solve carries NaN, and every window of a
    batch is bit for bit its one-window solve (NaN by position)."""
    inp = stage_inputs()
    t_cond = torch.atan(inp["cond_snr"])
    cond_inputs = [v.view(-1) for v in torch.log(torch.tan(t_cond) / 8.0)]
    sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
    ctxs = [(0, 0, 0), (0, 1, -2), (0, -1, 3)]
    maps = []
    for i, _ in enumerate(ctxs):
        mp = inp["coarse_map"].clone() * (1 + 0.1 * i)
        if i == 1:
            mp[0, 30:33, 40] = NAN                  # nodata cells of an imported raster
            mp[3, 5, 60] = NAN
        maps.append(mp)
    ww = linear_weight_window(64)
    args = (t_cond, cond_inputs, ww, inp["coarse_means"].tolist(), inp["coarse_stds"].tolist())
    batch = coarse_stage_tiles(coarse_model, sched, SEED, ctxs, maps, *args)
    for i, (ctx, mp) in enumerate(zip(ctxs, maps)):
        one = coarse_stage_tile(coarse_model, sched, SEED, ctx, mp, *args)
        NF.assert_same_bits(batch[i], one, f"window {ctx}")
        has_nan = bool(torch.isnan(one[:-1]).any())
        assert has_nan == (i == 1), f"window {ctx}: NaN {'missing' if i == 1 else 'leaked in'}"


# ------------------------------------------------------------------------------------------------ against the reference
G_NAN = np.load(Path(__file__).resolve().parent / "golden" / "coarse_nan_golden.npz")


def _stage_args():
    inp = stage_inputs()
    t_cond = torch.atan(inp["cond_snr"])
    cond_inputs = [v.view(-1) for v in torch.log(torch.tan(t_cond) / 8.0)]
    return inp, (t_cond, cond_inputs, linear_weight_window(64), inp["coarse_means"].tolist(),
                 inp["coarse_stds"].tolist())


def test_coarse_stage_matches_the_reference_on_nan_conditioning_cells(coarse_model):
    """The reference's own _coarse_inference on a window with NaN cells (tests/golden/make_golden_coarse_nan.py):
    NaN in exactly its positions, the finite elements (the blend weights) bit for bit, and the same window without the
    NaN cells to the stage tolerance."""
    inp, args = _stage_args()
    sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
    want = torch.from_numpy(G_NAN["nan"])
    assert bool(torch.isnan(want).any())
    got = coarse_stage_tile(coarse_model, sched, SEED, NF.COARSE_NAN_CTX, NF.coarse_nan_map(inp["coarse_map"]),
                            *args).cpu()
    finite = NF.assert_same_nonfinite(got, want, "coarse window with NaN cells")
    assert torch.equal(got[finite], want[finite])
    batch = coarse_stage_tiles(coarse_model, sched, SEED, [(0, 0, 0), NF.COARSE_NAN_CTX],
                               [inp["coarse_map"], NF.coarse_nan_map(inp["coarse_map"])], *args)
    NF.assert_same_bits(batch[1], got, "the window in a batch")
    assert bool(torch.isfinite(batch[0]).all())
    clean = coarse_stage_tile(coarse_model, sched, SEED, NF.COARSE_NAN_CTX, inp["coarse_map"].clone(), *args).cpu()
    assert IR.rel_rms(clean[:-1], torch.from_numpy(G_NAN["clean"])[:-1]) < 1.0e-2


def test_world_pipeline_carries_nan_conditioning_to_the_coarse_canvas_and_gets_finite_terrain():
    """A WorldPipeline whose conditioning_fn gives window (1, -2) the NaN cells of the golden: its coarse canvas carries
    NaN over that window's footprint, where the reference's does, and get() over it is finite terrain (the latent
    stage replaces NaN by the conditioning mean, world_pipeline.py:1018-1050)."""
    inp, _ = _stage_args()
    y0, x0 = NF.COARSE_NAN_CTX[1] * 48, NF.COARSE_NAN_CTX[2] * 48

    def cond_fn(i1, i2, j1, j2):
        if (i1, i2, j1, j2) == (y0, y0 + 64, x0, x0 + 64):
            return NF.coarse_nan_map(inp["coarse_map"])
        g = torch.Generator().manual_seed((i1 * 7919 + j1) % (1 << 31))
        return torch.randn(5, i2 - i1, j2 - j1, generator=g)

    models = []
    for name in ("coarse", "base", "decoder"):
        m = EDMUnet2D(**CONFIGS[name]).eval()
        m.load_state_dict(ounet.procedural_state_dict(CONFIGS[name], seed=0))
        models.append(m)
    world = WorldPipeline.from_local_models(*models, seed=5, decoder_tile_size=128, decoder_tile_stride=96,
                                            residual_mean=0.1, residual_std=1.2, conditioning_fn=cond_fn).to("cuda").bind()
    canvas = world.coarse[:, y0 - 8:y0 + 72, x0 - 8:x0 + 72]
    want = torch.zeros_like(canvas, dtype=torch.bool)
    want[:6, 8:72, 8:72] = torch.from_numpy(np.isnan(G_NAN["nan"][:6]))     # every data channel of the footprint
    assert torch.equal(torch.isnan(canvas), want)
    # pixels (128 per coarse cell) inside the footprint, across its border and outside it
    for ci, cj in ((y0 + 32, x0 + 32), (y0, x0 + 63), (y0 - 40, x0 - 40)):
        out = world.get(ci * 128, cj * 128, ci * 128 + 64, cj * 128 + 64)
        assert torch.isfinite(out["elev"]).all() and torch.isfinite(out["climate"]).all(), (ci, cj)
