"""The non-finite references of tests/_nonfinite.py are honest: on small random cases, the NaN mask of each fp64
reference equals the structural taint map (which outputs a poisoned input can reach through 3x3 support, the pixel
norm, attention and resampling), and the comparison helpers fail where they should.  No GPU needed."""
from __future__ import annotations

import dataclasses

import pytest
import torch

from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from tests import _igemm_ref as IR
from tests import _nonfinite as NF
from tests.test_oracle_golden import TINY_CFGS

NAN = float("nan")
E, R, P = L.EPI_EMB_SILU, L.EPI_RESID, L.EPI_PNORM

CASES = [
    IR.Case("3x3", [(8, 9)], 16, 3, 16, 16),
    IR.Case("1x1_pnorm", [(8, 1)], 16, 2, 16, 8, epi=P, outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_SILU, L.SP_SAME, 1.0)]),
    IR.Case("emb_silu_clip", [(8, 9)], 8, 2, 16, 16, epi=E, clip=0.5),
    IR.Case("3seg_resid_pnorm", [(8, 9), (16, 1), (8, 1)], 8, 2, 16, 16, epi=R, resid_pnorm=1, clip=0.4,
            outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_DOWN2, 1.0), (L.OUT_SILU, L.SP_UP2, 0.8)]),
    IR.Case("resid_up", [(8, 9)], 8, 2, 16, 16, epi=R, resid_spatial=L.SP_UP2, rms_out=True,
            outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_SAME, 1.0)]),
    IR.Case("resid_down_pnorm", [(8, 9)], 8, 3, 16, 16, epi=R | P, resid_spatial=L.SP_DOWN2, resid_pnorm=1),
]


def _poison(t: torch.Tensor, pixels, channel=None):
    """NaN at (image, y, x) of each pixel: one channel, or all of them."""
    t = t.clone()
    for n, y, x in pixels:
        if channel is None:
            t[n, :, y, x] = NAN
        else:
            t[n, channel, y, x] = NAN
    return t


def _pixel_map(shape, pixels):
    m = torch.zeros(shape[0], 1, *shape[2:], dtype=torch.bool)
    for n, y, x in pixels:
        m[n, 0, y, x] = True
    return m


def _assert_mask(ref, taint, what):
    want = taint.expand_as(ref) if ref.dim() == 4 else taint
    got = torch.isnan(ref)
    assert torch.equal(got, want), f"{what}: {int((got != want).sum())} elements differ from the taint map"


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("where", ["a", "resid", "cvec"])
def test_igemm_reference_nan_mask_is_the_taint_map(case, where):
    acts, wts, cvec, resid = IR.make_inputs(case, "cpu")
    n, h, w = case.n, case.h, case.w
    rh, rw = resid.shape[2:]
    a_t = [torch.zeros(n, 1, h, w, dtype=torch.bool) for _ in acts]
    r_t, c_t = torch.zeros(n, 1, rh, rw, dtype=torch.bool), torch.zeros(n, dtype=torch.bool)
    if where == "a":
        px = [(0, 0, 0), (0, h // 2, w // 2 - 1), (n - 1, h - 1, w // 2)]
        acts = [_poison(acts[-1], px, channel=1) if i == len(acts) - 1 else a for i, a in enumerate(acts)]
        a_t[-1] = _pixel_map(acts[-1].shape, px)
    elif where == "resid":
        if not case.epi & R:
            pytest.skip("no residual")
        px = [(0, rh - 1, 0), (n - 1, rh // 2, rw // 2)]
        resid = _poison(resid, px)
        r_t = _pixel_map(resid.shape, px)
    else:
        if not case.epi & E:
            pytest.skip("no modulation vector")
        cvec = cvec.clone()
        cvec[n - 1, :] = NAN
        c_t[n - 1] = True
    refs = NF.igemm_reference(case, acts, wts, cvec, resid)
    taints = NF.taint_igemm(case, a_t, r_t, c_t)
    assert len(refs) == len(taints)
    for i, (ref, t) in enumerate(zip(refs, taints)):
        _assert_mask(ref, t, f"{case.name} out{i}")
        assert bool(torch.isnan(ref).any())


def test_one_nan_residual_channel_spreads_only_through_the_pixel_norm():
    case = dataclasses.replace(CASES[3], resid_pnorm=0, clip=0.0)
    acts, wts, cvec, resid = IR.make_inputs(case, "cpu")
    resid = _poison(resid, [(1, 2, 4)], channel=2)
    raw, pnorm_silu, _ = NF.igemm_reference(case, acts, wts, cvec, resid)
    assert torch.isnan(raw).sum() == 1 and bool(torch.isnan(raw[1, 2, 2, 4]))
    assert bool(torch.isnan(pnorm_silu[1, :, 1, 2]).all()) and torch.isnan(pnorm_silu).sum() == case.cout


def test_resid_inv_reference_keeps_nan():
    case = dataclasses.replace(CASES[3], resid_inv=True)
    acts, wts, cvec, resid = IR.make_inputs(case, "cpu")
    inv = 1.0 / (1e-4 + resid.double().square().mean(dim=1).sqrt())
    inv[0, 4, 4] = NAN
    raw = NF.igemm_reference(case, acts, wts, cvec, resid, resid_inv=inv)[0]
    assert bool(torch.isnan(raw[0, :, 4, 4]).all()) and torch.isnan(raw).sum() == case.cout
    clean = NF.igemm_reference(case, acts, wts, cvec, resid, resid_inv=inv.nan_to_num(1.0))[0]
    want = IR.reference(case, acts, wts, cvec, resid)[0]
    keep = torch.ones_like(raw, dtype=torch.bool)
    keep[0, :, 4, 4] = False
    assert torch.allclose(clean[keep], want[keep], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("which", ["q", "k", "v"])
def test_attention_reference_nan_mask(which):
    g = torch.Generator().manual_seed(5)
    n, heads, tokens = 3, 2, 12
    q, k, v = (torch.randn(n, heads * 64, tokens, generator=g) for _ in range(3))
    t = {"q": q, "k": k, "v": v}[which]
    t[1, 64 + 7, 5] = NAN                     # image 1, head 1, one channel of token 5
    out = NF.attention_reference(q, k, v, heads).reshape(n, heads, 64, tokens)
    nan = torch.isnan(out)
    want = torch.zeros_like(nan)
    if which == "q":
        want[1, 1, :, 5] = True               # a NaN query poisons only its own row
    else:
        want[1, 1] = True                     # a NaN key or value poisons every query of its head
    assert torch.equal(nan, want)


def test_attention_reference_turns_inf_into_nan():
    g = torch.Generator().manual_seed(6)
    q, k, v = (torch.randn(1, 64, 8, generator=g) for _ in range(3))
    q[0, 3, 2] = float("inf")
    out = NF.attention_reference(q, k, v, 1)
    assert bool(torch.isnan(out[0, :, 2]).all()) and torch.isnan(out).sum() == 64   # x / (eps + rms) = inf / inf


@pytest.mark.parametrize("name,hw,pixels", [
    ("tiny_dec", 32, [(0, 0, 0)]),
    ("tiny_dec", 64, [(1, 40, 21)]),
    ("tiny_attn_cond", 16, [(0, 15, 3)]),
])
def test_unet_forward_nan_mask_is_the_taint_map(name, hw, pixels):
    cfg = TINY_CFGS[name]
    sd = {k: v.double() if v.is_floating_point() else v for k, v in ounet.procedural_state_dict(cfg, seed=3).items()}
    g = torch.Generator().manual_seed(13)
    n = 3
    x = torch.randn(n, cfg["in_channels"], hw, hw, generator=g, dtype=torch.float64)
    t = torch.rand(n, generator=g, dtype=torch.float64)
    cond = []
    for kind, dim, _ in cfg.get("conditional_inputs") or []:
        if kind == "tensor":
            cond.append(torch.randn(n, dim, generator=g, dtype=torch.float64))
        elif kind == "float":
            cond.append(torch.randn(n, generator=g, dtype=torch.float64))
        else:
            cond.append(torch.randint(0, dim, (n,), generator=g))
    x = _poison(x, pixels, channel=cfg["in_channels"] - 1)
    y = ounet.unet_forward(sd, cfg, x, t, cond)
    taint = NF.taint_forward(cfg, sd, _pixel_map(x.shape, pixels))
    _assert_mask(y, taint, name)
    assert bool(torch.isnan(y).any()) and not bool(torch.isnan(y[[i for i in range(n) if i not in
                                                                    {p[0] for p in pixels}]]).any())


def test_comparison_helpers_fail_where_they_should():
    ref = torch.tensor([1.0, NAN, float("inf"), -float("inf"), -2.0], dtype=torch.float64)
    NF.assert_matches(ref.float().bfloat16(), ref, "same")
    for bad in ([1.0, 0.0, float("inf"), -float("inf"), -2.0],           # NaN lost
                [1.0, NAN, NAN, -float("inf"), -2.0],                     # +inf became NaN
                [1.0, NAN, float("inf"), float("inf"), -2.0],             # -inf flipped
                [NAN, NAN, float("inf"), -float("inf"), -2.0],            # extra NaN
                [1.1, NAN, float("inf"), -float("inf"), -2.0]):           # finite element out of bound
        with pytest.raises(AssertionError):
            NF.assert_matches(torch.tensor(bad), ref, "bad")
    NF.assert_same_bits(torch.tensor([1.0, NAN, 3.0]), torch.tensor([1.0, -NAN, 3.0]), "payload")
    with pytest.raises(AssertionError):
        NF.assert_same_bits(torch.tensor([1.0, NAN, 3.0]), torch.tensor([1.0, NAN, 3.0000002]), "bits")
