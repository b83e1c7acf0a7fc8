"""NaN and +-inf through the U-Net path: a comparison that keeps non-finite values, an fp64 reference that keeps them,
and a structural taint map that says which outputs a poisoned input can reach.

The references are the existing ones run in fp64 on the CPU (tests/_igemm_ref.reference, oracle/unet.py): torch.clip,
softmax, the pixel norm and mp_silu keep NaN there by construction.  fp32 CPU convolution is not used: oneDNN may pick
Winograd for a 3x3, and Winograd spreads a NaN over a whole transform tile.

NaN payload and sign are not compared: the device's canonical NaN is not x86's.
"""
from __future__ import annotations

import dataclasses

import torch
import torch.nn.functional as F

from oracle import unet as ounet
from tests import _igemm_ref as IR

NAN, INF = float("nan"), float("inf")


def _first(mask: torch.Tensor) -> tuple:
    return tuple(int(v) for v in mask.nonzero()[0])


def assert_same_nonfinite(got: torch.Tensor, ref: torch.Tensor, what: str) -> torch.Tensor:
    """NaN, +inf and -inf of `got` in exactly the positions of `ref`.  Returns the mask of ref's finite elements."""
    got, ref = got.double().cpu(), ref.double().cpu()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    for name, f in (("NaN", torch.isnan), ("+inf", lambda t: t == INF), ("-inf", lambda t: t == -INF)):
        g, r = f(got), f(ref)
        bad = g != r
        if bool(bad.any()):
            raise AssertionError(f"{what}: {name} at {int(bad.sum())} positions that differ from the reference "
                                 f"(got {int(g.sum())}, want {int(r.sum())}; first {_first(bad)})")
    return torch.isfinite(ref)


def finite_ratio(got: torch.Tensor, ref: torch.Tensor, finite: torch.Tensor) -> float:
    """elementwise_ratio of tests/_igemm_ref.py over the finite elements only: max |got - ref| / (2^-7 |ref| +
    2^-12 rms(ref)), the rms taken over ref's finite elements."""
    if not bool(finite.any()):
        return 0.0
    g, r = got.double().cpu()[finite], ref.double().cpu()[finite]
    bound = 2.0 ** -7 * r.abs() + 2.0 ** -12 * float(r.square().mean().sqrt())
    return float(((g - r).abs() / bound).max())


def assert_matches(got, ref, what, limit: float = 1.0) -> float:
    """Non-finite positions exact, every finite element within `limit` x the per-element bound of finite_ratio."""
    finite = assert_same_nonfinite(got, ref, what)
    ratio = finite_ratio(got, ref, finite)
    assert ratio <= limit, f"{what}: error {ratio:.2f}x the per-element bound"
    return ratio


def finite_rel_rms(got, ref, finite) -> float:
    if not bool(finite.any()):
        return 0.0
    return IR.rel_rms(got.double().cpu()[finite], ref.double().cpu()[finite])


def assert_same_bits(got: torch.Tensor, want: torch.Tensor, what: str):
    """Bit for bit, except that NaN is compared by position only."""
    assert_same_nonfinite(got, want, what)
    g, w = got.cpu(), want.cpu()
    keep = ~torch.isnan(w)
    assert torch.equal(g[keep], w[keep]), f"{what}: finite bits differ"


# ------------------------------------------------------------------------------------------------ fp64 references
def igemm_reference(case: IR.Case, acts, wts, cvec, resid, resid_inv=None, device="cpu") -> list:
    """tests/_igemm_ref.reference in fp64.  resid_inv: the residual's pixel-norm factor plane the launch reads instead
    of recomputing it (case.resid_inv), NaN and all.  On a CUDA device cuDNN is switched off, so the convolution is
    torch's own im2col + GEMM: no transform algorithm that would spread a NaN beyond the 3 x 3 support."""
    dev = torch.device(device)
    args = [t.to(dev) for t in acts], [t.to(dev) for t in wts], cvec.to(dev), resid.to(dev).double()
    if resid_inv is not None and case.epi & IR.L.EPI_RESID:
        case = dataclasses.replace(case, resid_pnorm=0)
        args = args[:3] + (args[3] * resid_inv.to(dev).double()[:, None],)
    with torch.backends.cudnn.flags(enabled=False):
        return IR.reference(case, *args)


def attention_reference(q, k, v, heads: int):
    """The cosine attention core of tests/test_direct_kernels_gpu.py in fp64: q, k, v [n, heads * 64, tokens]."""
    n, c, tokens = q.shape

    def norm(t):
        t = t.double().cpu().reshape(n, heads, 64, tokens)
        return t / (1e-4 + t.square().mean(dim=2, keepdim=True).sqrt())

    qn, kn, vn = norm(q), norm(k), norm(v)
    w = torch.softmax(torch.einsum("nhdq,nhdk->nhqk", qn, kn) / 8.0, dim=-1)
    return torch.einsum("nhqk,nhdk->nhdq", w, vn).reshape(n, c, tokens)


# ------------------------------------------------------------------------------------------------ taint maps
# A taint map is a bool [n, 1, h, w] pixel mask (every op below mixes all channels of a pixel, so one plane is enough):
# the pixels a NaN input can reach.
def taint_pixels(x: torch.Tensor) -> torch.Tensor:
    """The NaN pixels of an activation [n, c, h, w]: any channel."""
    return torch.isnan(x).any(dim=1, keepdim=True)


def taint_conv(t: torch.Tensor, k: int) -> torch.Tensor:
    """A k x k convolution (k = 1 or 3, zero padding): every output pixel whose support holds a tainted pixel."""
    if k == 1:
        return t
    return F.max_pool2d(t.float(), 3, stride=1, padding=1) > 0


def taint_resample(t: torch.Tensor, mode: str) -> torch.Tensor:
    return ounet.resample(t, mode)


def taint_attention(t: torch.Tensor) -> torch.Tensor:
    """Cosine attention over the tokens of one image: a tainted key or value reaches every query, a tainted query its
    own row, so any tainted token taints the whole image."""
    return t.flatten(1).any(dim=1)[:, None, None, None].expand_as(t)


def taint_block(t: torch.Tensor, b: dict, has_skip: bool, heads: int) -> torch.Tensor:
    """oracle.unet.unet_block: resample, 1x1 skip, pixel norm (per pixel), conv_res0 / conv_res1 (3 x 3), mp_sum,
    attention, clip (per element)."""
    t = taint_resample(t, b["resample"])
    y = taint_conv(taint_conv(t, 3), 3)
    x = t | y
    if b.get("attention") and heads:
        x = x | taint_attention(x)
    return x


def taint_forward(cfg: dict, sd: dict, t: torch.Tensor) -> torch.Tensor:
    """oracle.unet.unet_forward on a taint map of its input x (the embedding untainted): the output pixels a NaN input
    pixel reaches."""
    enc, dec = ounet.block_plan(cfg)
    cph = (cfg.get("block_kwargs") or {}).get("channels_per_head", 64)
    skips = []
    for b in enc:
        if b["kind"] == "conv":
            t = taint_conv(t, sd[f"enc.{b['name']}.weight"].shape[-1])
        else:
            t = taint_block(t, b, f"enc.{b['name']}.conv_skip.weight" in sd, b["cout"] // cph)
        skips.append(t)
    for b in dec:
        if b.get("concat"):
            t = t | skips.pop()
        t = taint_block(t, b, f"dec.{b['name']}.conv_skip.weight" in sd, b["cout"] // cph)
    return taint_conv(t, sd["out_conv.weight"].shape[-1])


def taint_igemm(case: IR.Case, a_taint: list, resid_taint: torch.Tensor | None, cvec_taint=None) -> list:
    """One igemm launch (tests/_igemm_ref.reference) on taint maps: the segments' convolutions, the emb-silu modulation
    (a tainted cvec entry of an image taints all its pixels: every pixel reads it), the residual (resampled), clip,
    pixel norm, the outputs' resampling.  Returns one map per output (and the rms plane with case.rms_out)."""
    t = None
    for (c, taps), at in zip(case.segs, a_taint):
        y = taint_conv(at, 3 if taps == 9 else 1)
        t = y if t is None else t | y
    if cvec_taint is not None and case.epi & IR.L.EPI_EMB_SILU:
        t = t | cvec_taint[:, None, None, None].expand_as(t)
    if resid_taint is not None and case.epi & IR.L.EPI_RESID:
        r = resid_taint
        if case.resid_spatial == IR.L.SP_UP2:
            r = taint_resample(r, "up")
        elif case.resid_spatial == IR.L.SP_DOWN2:
            r = taint_resample(r, "down")
        t = t | r
    outs = []
    for kind, spatial, _ in case.outs:
        o = t
        if spatial == IR.L.SP_DOWN2:
            o = taint_resample(o, "down")
        elif spatial == IR.L.SP_UP2:
            o = taint_resample(o, "up")
        outs.append(o)
    if case.rms_out:
        outs.append(t[:, 0])
    return outs


# ------------------------------------------------------------------------------------------------ coarse window
COARSE_NAN_CTX = (0, 1, -2)


def coarse_nan_map(coarse_map: torch.Tensor) -> torch.Tensor:
    """The raw [5, 64, 64] coarse conditioning with NaN (nodata) cells in two channels, one at the window's border:
    what an imported raster with holes or a conditioning_fn gives the coarse stage."""
    m = coarse_map.clone()
    m[0, 30:33, 40] = float("nan")
    m[3, 5, 63] = float("nan")
    return m
