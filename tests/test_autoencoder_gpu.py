"""EDMAutoencoder and its tiled samplers on the GPU: against the reference's goldens (tests/golden/autoencoder_golden.npz,
written by tests/golden/make_golden_autoencoder.py), against the fp32 oracle at the benchmark shapes, and every
implicit-GEMM plan class the encoder and decoder launch there against fp64 (tests/_igemm_ref.py).

Tolerance (DESIGN section 2): rel-RMS <= 1.0e-2 vs the reference's fp32 output AND <= 1.25 x the reference's own
bf16-autocast error on the same inputs; where that error alone exceeds 1.0e-2 (every case here), only the second half
applies.  Each check prints its error share of the binding bound.
"""
from __future__ import annotations

import collections
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import autoencoder as oae
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import decode_autoencoder_latents_tiled, sample_autoencoder_tiled
from terrain_diffusion_b200.layout import from_nc8hw8
from terrain_diffusion_b200.models import EDMAutoencoder
from terrain_diffusion_b200.models.plan import FoldedWeights, autoencoder_decoder_plan
from tests._igemm_ref import case_from_desc, check_case, plan_class, plan_label, plan_of, report
from tests.test_autoencoder_cpu import _record
from tests._igemm_surface import representatives

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "autoencoder_golden.npz")
CFG = oae.X8_CFG
BENCH_TILES, BENCH_TILE = 8, 512      # tools/bench_autoencoder.py


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def check(y, ref, ref_err, what):
    err = rel_rms(y.float().cpu(), ref)
    assert float(ref.std()) > 0.01
    bound = 1.25 * ref_err if ref_err > 1.0e-2 else min(1.0e-2, 1.25 * ref_err)
    print(f"\n{what}: rel-RMS {err:.3e}, reference bf16 {ref_err:.3e}, share of bound {err / bound:.3f}")
    assert err <= bound, (what, err, ref_err)


def golden(name):
    return torch.from_numpy(G[name])


def check_golden(y, case):
    check(y, golden(f"{case}.y"), float(G[f"{case}.ref_bf16_err"]), case)


@pytest.fixture(scope="module")
def model():
    m = EDMAutoencoder(**CFG).eval()
    m.load_state_dict(oae.procedural_state_dict(CFG, seed=0))
    return m.cuda()


def test_goldens_through_the_public_calls(model):
    means, logvars = model.preencode(golden("enc.x").cuda())
    assert means.shape == logvars.shape == (2, 4, 8, 8)
    check(torch.cat([means, logvars], dim=1), torch.cat([golden("enc.means"), golden("enc.logvars")], dim=1),
          float(G["enc.ref_bf16_err"]), "enc")
    check_golden(model.decode(golden("dec.z").cuda()), "dec")
    check_golden(sample_autoencoder_tiled(model, golden("rec96.images").cuda(), 64, 32, use_mode=True), "rec96")
    check_golden(decode_autoencoder_latents_tiled(model, golden("dec96.latents").cuda(), 64, 32), "dec96")
    enc = model.encoder(golden("enc.x").cuda(), None)          # EDMUnet2D(encode_only=True): out_conv at 1/8
    assert torch.equal(enc, torch.cat([means, logvars], dim=1))


def test_tile_batch_meets_the_same_golden_and_repeats_bit_identically(model):
    img, lat = golden("rec96.images").cuda(), golden("dec96.latents").cuda()
    for tb in (1, 2, None):
        rec = sample_autoencoder_tiled(model, img, 64, 32, use_mode=True, tile_batch=tb)
        check_golden(rec, "rec96")
        assert torch.equal(rec, sample_autoencoder_tiled(model, img, 64, 32, use_mode=True, tile_batch=tb))
        dec = decode_autoencoder_latents_tiled(model, lat, 64, 32, tile_batch=tb)
        check_golden(dec, "dec96")
        assert torch.equal(dec, decode_autoencoder_latents_tiled(model, lat, 64, 32, tile_batch=tb))


def test_sampling_draws_each_tile_in_row_major_order(model):
    """use_mode=False: tile_batch does not change which draw a tile's latent gets (one randn_like per tile, row-major),
    and the result equals the oracle's blend with those draws to the bf16 bound."""
    img = golden("rec96.images").cuda()
    outs = []
    for tb in (1, None):
        torch.cuda.manual_seed(11)
        outs.append(sample_autoencoder_tiled(model, img, 64, 32, tile_batch=tb))
    torch.cuda.manual_seed(11)
    eps = [torch.randn(1, 4, 8, 8, device="cuda").cpu() for _ in range(4)]
    ref = oae.sample_autoencoder_tiled(oae.procedural_state_dict(CFG, seed=0), CFG, golden("rec96.images"), 64, 32,
                                       eps=eps)
    for out in outs:
        check(out, ref, float(G["rec96.ref_bf16_err"]), "rec96 sampled")


@pytest.mark.parametrize("ch,hw", [(1, (40, 24)), (4, (16, 8)), (1, (64, 64)), (4, (8, 8))])
def test_im2col_of_the_autoencoder_first_convolutions_is_exact(ch, hw):
    """tdx_im2col_run <2> (encoder: image + ones) and <5> (decoder: 4 latents + ones): channel k = tap*ci + c of the
    zero-padded 3x3 neighbourhoods, exact up to the single bf16 rounding of each value."""
    dev = torch.device("cuda:0")
    h, w = hw
    n = 2
    src = torch.randn(n, ch, h, w, generator=torch.Generator().manual_seed(5)).to(dev)
    scale = torch.tensor([0.37], device=dev)
    ci = ch + 1
    out = torch.full((n, 8, h, w, 8), float("nan"), dtype=torch.bfloat16, device=dev)
    d = L.TdxIm2colDesc()
    d.src[0], d.src_channels[0], d.src_dtype[0], d.src_scale[0] = src.data_ptr(), ch, 0, scale.data_ptr()
    d.out, d.k_pad = out.data_ptr(), 64
    d.n_img, d.height, d.width = n, h, w
    L.check(L.lib().tdx_im2col_run(C.byref(d), L.current_stream_ptr()))
    torch.cuda.synchronize()
    x = torch.cat([src * scale, torch.ones(n, 1, h, w, device=dev)], dim=1)
    cols = F.unfold(x, kernel_size=3, padding=1).view(n, ci, 9, h, w)
    ref = cols.permute(0, 2, 1, 3, 4).reshape(n, 9 * ci, h, w).bfloat16().float()
    got = from_nc8hw8(out)
    assert torch.equal(got[:, :9 * ci], ref)
    assert torch.count_nonzero(got[:, 9 * ci:]) == 0


def test_centre_tap_first_convolution_equals_the_1x1_decoder_conv(model):
    """The decoder's first launch pair (im2col <5> + 1x1 igemm over the centre-tap weight matrix) against the 1x1
    decoder_conv over [z, ones] in fp64 on the same bf16 operands: only the bf16 rounding of the stored output."""
    z = torch.randn(2, 4, 16, 24, generator=torch.Generator().manual_seed(9)).cuda()
    model.decode(z)
    prog, _ = model._plans[("dec", 2, 16, 24)]
    got = from_nc8hw8(prog.arena["enc.conv..raw"]).double()
    fw = model.folded()
    w = fw.segs["conv_in.im2col"][0][:, 4 * 5:5 * 5, 0, 0].bfloat16().double().cuda()     # centre tap, [256][5]
    x = torch.cat([z, torch.ones_like(z[:, :1])], dim=1).bfloat16().double()
    ref = F.conv2d(x, w[:, :, None, None])
    assert float((got - ref).abs().max()) <= 2 ** -8 * float(ref.abs().max())
    assert rel_rms(got, ref) < 2e-3


@pytest.fixture()
def fp32_oracle_on_gpu():
    """The oracle in true fp32 on the device (no TF32) for the 512^2 shapes, which are slow on the host."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield {k: v.cuda() for k, v in oae.procedural_state_dict(CFG, seed=0).items()}
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_benchmark_shapes_match_the_oracle(model, fp32_oracle_on_gpu):
    """A 512^2 encode at B=8 and a 64^2-latent decode at B=8, under the bound of the same call's golden."""
    sd = fp32_oracle_on_gpu
    g = torch.Generator().manual_seed(4)
    x = torch.randn(BENCH_TILES, 1, BENCH_TILE, BENCH_TILE, generator=g).cuda()
    means, logvars = model.preencode(x)
    rm, rl = oae.preencode(sd, CFG, x)
    check(torch.cat([means, logvars], dim=1), torch.cat([rm, rl], dim=1).cpu(), float(G["enc.ref_bf16_err"]),
          "enc 8x512^2")
    z = torch.randn(BENCH_TILES, 4, BENCH_TILE // 8, BENCH_TILE // 8, generator=g).cuda()
    check(model.decode(z), oae.decode(sd, CFG, z).cpu(), float(G["dec.ref_bf16_err"]), "dec 8x64^2 latents")


def test_postencode_is_the_reference_formula_bit_for_bit(model):
    means, logvars = model.preencode(golden("enc.x").cuda())
    torch.cuda.manual_seed(123)
    got = model.postencode(means, logvars)
    torch.cuda.manual_seed(123)
    std = torch.exp(logvars * 0.5)
    want = means + torch.randn_like(std) * std
    assert torch.equal(got, want)
    assert model.postencode(means, logvars, use_mode=True) is means


def test_save_and_from_pretrained_round_trip(model, tmp_path):
    model.save_pretrained(tmp_path)
    back = EDMAutoencoder.from_pretrained(tmp_path).cuda()
    assert dict(back.config) == dict(model.config)
    z = golden("dec.z").cuda()
    assert torch.equal(back.decode(z), model.decode(z))
    x = golden("enc.x").cuda()
    assert all(torch.equal(a, b) for a, b in zip(back.preencode(x), model.preencode(x)))
    out, logvar = back.decode(z, include_logvar=True)
    assert logvar.shape == (1, 1, 1, 1)


def _autoencoder_launches():
    """[(source, case, plan)] for every igemm launch of the encoder and decoder at the benchmark shapes."""
    m = EDMAutoencoder(**CFG).eval()
    meta = torch.device("meta")
    progs = [("encode", _record(FoldedWeights(m.encoder, meta), BENCH_TILES, BENCH_TILE, BENCH_TILE, 1, True)[0]),
             ("decode", _record(FoldedWeights(m.decoder_view(), meta, plan=autoencoder_decoder_plan(m._decoder_config())),
                                BENCH_TILES, BENCH_TILE // 8, BENCH_TILE // 8, 4, False)[0])]
    out = []
    for source, prog in progs:
        for d in prog.igemm():
            c = case_from_desc(d, name=f"{source}:{prog.key_of.get(d.out[0].ptr, '?')}")
            out.append((source, None, c, plan_of(c)))
    return out


def test_every_autoencoder_plan_class_matches_fp64(request):
    """The smallest launch of every (plan class, epilogue signature) group of the benchmark-shape encoder and decoder
    is replayed against fp64; one line per plan class is written to the terminal."""
    launches = _autoencoder_launches()
    reps = representatives(launches)
    margins: dict = {}
    for c in reps:
        check_case(c, torch.device("cuda:0"), margins)
    per_class = collections.Counter(plan_class(p) for _, _, _, p in launches)
    covered = {}
    for c in reps:
        covered.setdefault(plan_class(plan_of(c)), c.name)
    worst = max(margins, key=margins.get)
    lines = [f"autoencoder: {len(per_class)} plan classes, {len(launches)} launches, {len(reps)} groups replayed; "
             f"worst per-element error {margins[worst]:.3f} of the bound ({worst})"]
    lines += [f"  {plan_label(cls):32s} launches={count:4d}  covered by {covered.get(cls, 'NOTHING')}"
              for cls, count in sorted(per_class.items())]
    report(request.config, lines)
    assert set(per_class) <= set(covered)
