"""FoldedWeights (models/plan.py) against the module math, without a GPU.

Every GEMM operand (`fw.segs`) and every fp32 table (`fw.g`) of the shipped models is recomputed here in fp64 straight
from the state dict: MPConv's weight normalisation (mp_layers.py:9-12, 203-213) restated below, and the mp_sum /
mp_concat constants taken from the oracle's own functions (oracle/unet.py) applied to ones, not from plan.py.  Bounds:

  per element   |fold - ref| <= (2^-8 + 2^-11) |ref| for the bf16 operands, 2^-11 |ref| for the fp32 tables;
  per tensor    the mean of fold / ref - 1 over the non-zero elements <= max(5e-4, 4 standard errors of that mean):
                bf16 rounding is unbiased, so a constant that is off by a fraction of a bf16 ulp still fails here.

The 2^-11 and 5e-4 are room for the fold's fp32 arithmetic: FoldedWeights normalises with an fp32 host norm, which is
off by up to 3.8e-4 on the 10.6 M elements of the base model's 1536 -> 768 3x3 weight (the whole layer scaled by that
much).  A constant off by 0.5 % still fails both bounds.

VARIANT_CFG is the base model with res_balance, attn_balance, clip_act and concat_balance all different from each
other and from the shipped 0.3 / 256 / 0.5, so a constant taken from the wrong place cannot pass by coincidence.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import pytest
import torch

from oracle import autoencoder as oae
from oracle import unet as ounet
from terrain_diffusion_b200.models import EDMAutoencoder, EDMUnet2D
from terrain_diffusion_b200.models.plan import FoldedWeights, autoencoder_decoder_plan
from tests._capture import CONFIGS

VARIANT_CFG = dict(CONFIGS["base"], concat_balance=0.35,
                   block_kwargs={"res_balance": 0.25, "attn_balance": 0.4, "clip_act": 1.5})
"""The base model with distinguishable mp_sum / mp_concat constants and a clip that is active at unit magnitudes."""
UNET_CONFIGS = dict(CONFIGS, variant=VARIANT_CFG)
MODELS = ["decoder", "base", "guide", "coarse", "variant", "ae_encoder", "ae_decoder"]
BF16_REL = 2.0 ** -8 + 2.0 ** -11
FP32_REL = 2.0 ** -11
MEAN_TOL = 5e-4


def block_kwargs(cfg: dict) -> dict:
    """oracle.unet.unet_block's keyword arguments for a model config (as oracle.unet.unet_forward reads them)."""
    bk = cfg.get("block_kwargs") or {}
    return dict(res_balance=bk.get("res_balance", 0.3), attn_balance=bk.get("attn_balance", 0.3),
                clip_act=bk.get("clip_act", 256.0), channels_per_head=bk.get("channels_per_head", 64))


def model_spec(name: str, device=torch.device("cpu")) -> SimpleNamespace:
    """One model with procedural weights, described the way the oracle sees it:
      model     the product module (EDMUnet2D, or the EDMAutoencoder for both ae_* entries)
      sd        the oracle's state dict (fp32, on `device`) in the names `first`, `out`, `blocks` use
      cfg       the oracle config (noise / conditional inputs, block constants)
      first     (state-dict key of the first convolution, [n, ci, h, w] is concatenated with ones)
      blocks    [(plan key prefix, state-dict prefix, oracle block dict)] in forward order; the block dicts of
                oracle.unet.block_plan / oracle.autoencoder.decoder_plan
      out       (out_conv key, out_gain)
      fold      () -> the product's FoldedWeights of this model on `device`."""
    if name.startswith("ae_"):
        cfg_ae = oae.X8_CFG
        sd_ae = oae.procedural_state_dict(cfg_ae, seed=0)
        m = EDMAutoencoder(**cfg_ae).eval()
        m.load_state_dict(sd_ae)
        if name == "ae_encoder":
            cfg = oae.encoder_config(cfg_ae)
            sd = {k[len("encoder."):]: v for k, v in sd_ae.items() if k.startswith("encoder.")}
            enc, _ = ounet.block_plan(cfg)
            return SimpleNamespace(
                model=m, sd={k: v.to(device) for k, v in sd.items()}, cfg=cfg, first=f"enc.{enc[0]['name']}.weight",
                blocks=[(f"enc.{b['name']}.", f"enc.{b['name']}.", b) for b in enc[1:]], enc=enc, dec=[],
                out=("out_conv.weight", sd["out_gain"]), fold=lambda: FoldedWeights(m.encoder, device))
        dec = oae.decoder_plan(cfg_ae)
        return SimpleNamespace(
            model=m, sd={k: v.to(device) for k, v in sd_ae.items()}, cfg=dict(cfg_ae, conditional_inputs=[]),
            first="decoder_conv.weight", blocks=[(f"dec.{i}.", f"decoder.{i}.", b) for i, b in enumerate(dec)],
            enc=None, dec=dec, out=("out_conv.weight", sd_ae["out_gain"]),
            fold=lambda: FoldedWeights(m.decoder_view(), device, plan=autoencoder_decoder_plan(m._decoder_config())))
    cfg = UNET_CONFIGS[name]
    sd = ounet.procedural_state_dict(cfg, seed=0)
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(sd)
    enc, dec = ounet.block_plan(cfg)
    blocks = [(f"enc.{b['name']}.", f"enc.{b['name']}.", b) for b in enc[1:]]
    blocks += [(f"dec.{b['name']}.", f"dec.{b['name']}.", b) for b in dec]
    return SimpleNamespace(model=m, sd={k: v.to(device) for k, v in sd.items()}, cfg=cfg,
                           first=f"enc.{enc[0]['name']}.weight", blocks=blocks, enc=enc, dec=dec,
                           out=("out_conv.weight", sd.get("out_gain", 1.0)), fold=lambda: FoldedWeights(m, device))


# ------------------------------------------------------------------------------------------------ fp64 restatement
def eff64(w: torch.Tensor, gain=1.0) -> torch.Tensor:
    """MPConv's effective weight in fp64: w / (1e-4 + ||w|| / sqrt(numel)) * gain / sqrt(fan_in)."""
    w = w.double()
    w = w / (1e-4 + torch.linalg.vector_norm(w) / math.sqrt(w.numel()))
    return w * (float(gain) / math.sqrt(w[0].numel()))


def mp_sum_weights(t: float) -> tuple[float, float]:
    """(weight of the first, weight of the second argument) of oracle.unet.mp_sum(., t), read off the oracle."""
    one, zero = torch.ones(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    return float(ounet.mp_sum([one, zero], t)), float(ounet.mp_sum([zero, one], t))


def mp_concat_weights(n_a: int, n_b: int, t: float) -> tuple[float, float]:
    """The two per-tensor scales of oracle.unet.mp_concat([a, b], t), read off the oracle."""
    y = ounet.mp_concat([torch.ones(1, n_a, dtype=torch.float64), torch.ones(1, n_b, dtype=torch.float64)], t)
    return float(y[0, 0]), float(y[0, n_a])


def expected_fold(spec) -> tuple[dict, dict]:
    """(segs, g) as FoldedWeights should hold them, in fp64."""
    sd, cfg = spec.sd, spec.cfg
    kw = block_kwargs(cfg)
    w_skip, w_res = mp_sum_weights(kw["res_balance"])
    _, w_attn = mp_sum_weights(kw["attn_balance"])
    cb = float(cfg.get("concat_balance", 0.3))
    cph = kw["channels_per_head"]
    segs, g = {}, {}
    # the first convolution: [cout][k_pad] with k = tap * ci + c, zero past 9 * ci; a 1x1 one sits on the centre tap
    w_in = eff64(sd[spec.first])
    cout, ci = w_in.shape[:2]
    k_pad = -(-9 * ci // 64) * 64
    mat = torch.zeros(cout, k_pad, dtype=torch.float64)
    for tap in range(9):
        ky, kx = divmod(tap, 3)
        if w_in.shape[-1] == 3:
            mat[:, tap * ci:(tap + 1) * ci] = w_in[:, :, ky, kx]
        elif tap == 4:
            mat[:, tap * ci:(tap + 1) * ci] = w_in[:, :, 0, 0]
    segs["conv_in.im2col"] = [mat[:, :, None, None]]
    # the last convolution: [tap][c][1 | 8], out_gain folded, zero past c_out
    w_out = eff64(sd[spec.out[0]], spec.out[1])
    co, c = w_out.shape[:2]
    wpad = 1 if co == 1 else 8
    tbl = torch.zeros(9, c, wpad, dtype=torch.float64)
    for tap in range(9):
        ky, kx = divmod(tap, 3)
        tbl[tap, :, :co] = w_out[:, :, ky, kx].t()
    g["conv_out"] = tbl
    # embedding layers (EDMUnet2D.compute_embeddings)
    if "noise_linear.weight" in sd:
        g["noise_linear"] = eff64(sd["noise_linear.weight"]).t()
        if cfg.get("fourier_scale", 1) == "pos":
            g["noise_freqs"] = sd["noise_fourier.freqs"].double()
    for i, (kind, _dim, _w) in enumerate(cfg.get("conditional_inputs") or []):
        if kind == "float":
            g[f"cond{i}"] = eff64(sd[f"conditional_layers.{i}.1.weight"]).t()
        elif kind == "tensor":
            g[f"cond{i}"] = eff64(sd[f"conditional_layers.{i}.weight"]).t()
        else:
            g[f"cond{i}"] = sd[f"conditional_layers.{i}.weight"].double()
    for key, p, b in spec.blocks:
        if p + "emb_linear.weight" in sd:
            g[key + "emb"] = eff64(sd[p + "emb_linear.weight"], sd[p + "emb_gain"]).t()
        w0 = eff64(sd[p + "conv_res0.weight"])
        w1 = eff64(sd[p + "conv_res1.weight"]) * w_res
        ws = eff64(sd[p + "conv_skip.weight"]) if p + "conv_skip.weight" in sd else None
        c = b["cout"]
        if b.get("attention") and c // cph:
            # attn_qkv output channel of (head, d, j) is head * 3 * cph + 3 * d + j (UNetBlock.attn's reshape)
            qkv = eff64(sd[p + "attn_qkv.weight"])
            ch = torch.arange(c)
            rows = (ch // cph) * 3 * cph + (ch % cph) * 3
            for j, nm in enumerate(("q", "k", "v")):
                segs[key + nm] = [qkv[rows + j]]
            segs[key + "proj"] = [eff64(sd[p + "attn_proj.weight"]) * w_attn]
        if b["mode"] == "enc":
            if ws is not None:
                segs[key + "k1"] = [ws]
            segs[key + "res0"] = [w0]
            segs[key + "res1"] = [w1]
        elif b.get("concat"):
            cx = b["cin"] - b["skip_channels"]
            s1, s2 = mp_concat_weights(cx, b["skip_channels"], cb)
            segs[key + "res0"] = [w0[:, :cx], w0[:, cx:]]
            segs[key + "res1"] = [w1, ws[:, :cx] * (s1 * w_skip), ws[:, cx:] * (s2 * w_skip)]
        else:
            segs[key + "res0"] = [w0]
            segs[key + "res1"] = [w1] + ([ws * w_skip] if ws is not None else [])
    return segs, g


def check_fold(got: torch.Tensor, ref: torch.Tensor, rel: float, what: str) -> float:
    """Per-element and per-tensor bounds of the module docstring; returns the worst per-element error / bound."""
    assert tuple(got.shape) == tuple(ref.shape), (what, tuple(got.shape), tuple(ref.shape))
    got, ref = got.double().cpu(), ref.double().cpu()
    err = (got - ref).abs()
    bound = rel * ref.abs()
    bad = err > bound
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {ref.numel()} elements outside {rel:.3g} x |ref| "
                                 f"(worst |err| / |ref| {float((err / ref.abs().clamp_min(1e-300)).max()):.3g})")
    nz = ref != 0
    if int(nz.sum()) > 1:
        r = got[nz] / ref[nz] - 1.0
        mean, se = float(r.mean()), float(r.std()) / math.sqrt(r.numel())
        assert abs(mean) <= max(MEAN_TOL, 4.0 * se), f"{what}: mean fold / ref - 1 = {mean:.3g} (standard error {se:.3g})"
    return float((err / bound.clamp_min(1e-300)).max()) if bool(nz.any()) else 0.0


@pytest.mark.parametrize("name", MODELS)
def test_folded_weights_equal_the_module_math(name):
    spec = model_spec(name)
    fw = spec.fold()
    # the scalars FoldedWeights reads from the config are the oracle's
    kw = block_kwargs(spec.cfg)
    assert (fw.t_res, fw.t_attn, fw.clip) == (kw["res_balance"], kw["attn_balance"], kw["clip_act"])
    if any(b.get("concat") for b in spec.dec):
        assert fw.cb == float(spec.cfg.get("concat_balance", 0.3))
    want_segs, want_g = expected_fold(spec)
    assert sorted(fw.segs) == sorted(want_segs)
    assert sorted(fw.g) == sorted(want_g)
    for key, parts in want_segs.items():
        got = fw.segs[key]
        assert len(got) == len(parts), (key, len(got), len(parts))
        for i, (a, b) in enumerate(zip(got, parts)):
            assert a.dtype == (torch.float32 if key == "conv_in.im2col" else torch.bfloat16), (key, a.dtype)
            check_fold(a, b, BF16_REL, f"{name} {key}[{i}]")
    for key, ref in want_g.items():
        assert fw.g[key].dtype == torch.float32, (key, fw.g[key].dtype)
        check_fold(fw.g[key], ref, FP32_REL, f"{name} g[{key}]")


def test_variant_constants_are_distinguishable():
    """The variant really separates the constants the planner could mix up (else the tests above cannot tell)."""
    kw = block_kwargs(VARIANT_CFG)
    ws, wr = mp_sum_weights(kw["res_balance"])
    wx, wa = mp_sum_weights(kw["attn_balance"])
    s1, s2 = mp_concat_weights(192, 192, VARIANT_CFG["concat_balance"])
    vals = [ws, wr, wx, wa, s1, s2]
    assert min(abs(a - b) for i, a in enumerate(vals) for b in vals[i + 1:]) > 0.05, vals
    assert kw["clip_act"] < 2.0
