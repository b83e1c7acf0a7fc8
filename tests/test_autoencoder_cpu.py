"""EDMAutoencoder without a GPU: parameter names against the reference class, the fp32 oracle against the reference's
goldens (tests/golden/autoencoder_golden.npz, written by tests/golden/make_golden_autoencoder.py), argument errors
before any CUDA call, and the encoder / decoder launch lists recorded on the meta device."""
from __future__ import annotations

import collections
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import autoencoder as oae
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import decode_autoencoder_latents_tiled, sample_autoencoder_tiled
from terrain_diffusion_b200.models import EDMAutoencoder
from terrain_diffusion_b200.models.plan import FoldedWeights, autoencoder_decoder_plan
from tests._capture import RecordingEmitter, RecordingProgram

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "autoencoder_golden.npz")
CFG = oae.X8_CFG
ENC_IGEMM = 25      # first conv + 2 per block + the 1x1 skip of 64->128 and 128->256
DEC_IGEMM = 35      # decoder_conv + 2 per block (17 blocks)
DEC_K_SLABS = 2     # 256->128 and 128->64: [h (3x3) | x (1x1)]


def max_rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("tag,extra", [("x8", {}), ("lpbd3", {"layers_per_block_decoder": 3})])
def test_state_dict_names_and_shapes_equal_the_reference_class(tag, extra):
    want = {n: tuple(int(v) for v in s.split("-") if v) for n, s in
            zip(G[f"shapes.{tag}.names"], G[f"shapes.{tag}.shapes"])}
    sd = EDMAutoencoder(**CFG, **extra).state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    assert oae.state_shapes(dict(CFG, **extra)) == want
    if tag == "x8":
        assert len(want) == 98 and EDMAutoencoder(**CFG).count_parameters() == 20_489_311


def test_oracle_matches_every_golden():
    sd = oae.procedural_state_dict(CFG, seed=0)
    means, logvars = oae.preencode(sd, CFG, torch.from_numpy(G["enc.x"]))
    assert max_rel(means, torch.from_numpy(G["enc.means"])) < 1e-5
    assert max_rel(logvars, torch.from_numpy(G["enc.logvars"])) < 1e-5
    assert max_rel(oae.decode(sd, CFG, torch.from_numpy(G["dec.z"])), torch.from_numpy(G["dec.y"])) < 1e-5
    rec = oae.sample_autoencoder_tiled(sd, CFG, torch.from_numpy(G["rec96.images"]), 64, 32)
    assert max_rel(rec, torch.from_numpy(G["rec96.y"])) < 1e-5
    dec = oae.decode_autoencoder_latents_tiled(sd, CFG, torch.from_numpy(G["dec96.latents"]), 64, 32)
    assert max_rel(dec, torch.from_numpy(G["dec96.y"])) < 1e-5
    for case in ("enc", "dec", "rec96", "dec96"):
        assert 0 < float(G[f"{case}.ref_bf16_err"]) < 0.05


@pytest.fixture()
def no_cuda(monkeypatch):
    """Any libtdx call or CUDA copy fails the test: the errors below must come first."""
    def boom(*_a, **_k):
        raise AssertionError("reached the device")
    monkeypatch.setattr(L, "lib", boom)
    monkeypatch.setattr(L, "call", boom)
    monkeypatch.setattr(torch.Tensor, "cuda", boom)


def test_argument_and_size_errors_come_before_any_cuda_call(no_cuda):
    m = EDMAutoencoder(**CFG).eval()
    with pytest.raises(ValueError, match="multiples of 64"):
        m.preencode(torch.zeros(1, 1, 96, 96))
    with pytest.raises(ValueError, match="multiples of 8"):
        m.decode(torch.zeros(1, 4, 12, 12))
    with pytest.raises(ValueError, match="multiples of 64"):
        sample_autoencoder_tiled(m, torch.zeros(1, 1, 96, 96), 48, 24)
    with pytest.raises(ValueError, match="fit"):
        sample_autoencoder_tiled(m, torch.zeros(1, 1, 64, 128))           # tile = width 128 > height 64
    with pytest.raises(ValueError, match="multiples of 8"):
        decode_autoencoder_latents_tiled(m, torch.zeros(1, 4, 12, 12))
    # stride 36: the tile at 36 decodes latents [4, 12) and keeps pixels 4..68 of 64 -- the reference's slice
    # assignment fails there with a shape mismatch
    with pytest.raises(ValueError, match="does not fit"):
        decode_autoencoder_latents_tiled(m, torch.zeros(1, 4, 16, 16), 64, 36)
    with pytest.raises(ValueError, match="does not fit"):
        decode_autoencoder_latents_tiled(m, torch.zeros(1, 4, 4, 4), 64, 32)  # 32^2 output < tile
    with pytest.raises(ValueError, match="multiples of 8"):
        decode_autoencoder_latents_tiled(m, torch.zeros(1, 4, 16, 16), 32, 16)  # 4^2 latent windows
    skips = EDMAutoencoder(**dict(CFG, direct_skips=[0])).eval()
    assert skips.state_dict()["decoder_conv.weight"].shape[1] == 6
    for call in (lambda: skips.preencode(torch.zeros(1, 1, 64, 64)), lambda: skips.decode(torch.zeros(1, 5, 8, 8)),
                 lambda: sample_autoencoder_tiled(skips, torch.zeros(1, 1, 64, 64)),
                 lambda: decode_autoencoder_latents_tiled(skips, torch.zeros(1, 5, 8, 8), 64)):
        with pytest.raises(NotImplementedError, match="direct_skips"):
            call()
    with pytest.raises(L.TdxError, match="inference-only"):
        m.train().decode(torch.zeros(1, 4, 8, 8))


def test_decode_geometry_follows_the_reference_slices():
    from terrain_diffusion_b200.inference.samplers import _latent_tile_geometry
    assert _latent_tile_geometry(12, 12, 64, 32) == [(i, j, i // 8, j // 8, 0, 0) for i in (0, 32) for j in (0, 32)]
    # tile 60 decodes 8 latents (64 pixels) and keeps 60 of them from offset i0 - 8 * (i0 // 8)
    assert _latent_tile_geometry(8, 8, 60, 4)[-1] == (4, 4, 0, 0, 4, 4)


def test_unsupported_input_channels_raise_before_device_work():
    with pytest.raises(NotImplementedError, match="over 2 input channels"):
        FoldedWeights(EDMAutoencoder(**dict(CFG, in_channels=2)).encoder, torch.device("meta"))


def _record(fw, n, h, w, c_in, with_embed):
    meta = torch.device("meta")
    prog = RecordingProgram()
    em = RecordingEmitter(fw, n, h, w, prog)
    if with_embed:
        em.emit_embed(prog, labels=torch.empty((n,), device=meta))
    em.emit(prog, [(torch.empty((n, c_in, h, w), device=meta), c_in, None)],
            model_out=torch.empty((n, fw.out_channels, em.out_h, em.out_w), device=meta))
    return prog, em


@pytest.mark.parametrize("n,hw", [(1, 64), (8, 512)])
def test_encoder_and_decoder_programs_are_recorded_without_a_gpu(n, hw):
    """One im2col each, no embed launch (emit_embed finds no modulated block), one conv_out, the expected igemm count;
    the decoder's channel-changing blocks carry conv_skip as a 1x1 K-slab of res1."""
    torch.manual_seed(0)
    m = EDMAutoencoder(**CFG).eval()
    meta = torch.device("meta")
    prog, em = _record(FoldedWeights(m.encoder, meta), n, hw, hw, 1, with_embed=True)
    kinds = collections.Counter(k for k, _ in prog.launches)
    assert kinds == collections.Counter(im2col=1, igemm=ENC_IGEMM, conv_out=1)
    assert (em.out_h, em.out_w) == (hw // 8, hw // 8)
    im = prog.launches[0][1]
    assert prog.launches[0][0] == "im2col" and im.k_pad == 64 and im.src_channels[0] == 1
    od = prog.launches[-1][1]
    assert od.c_out == 8 and od.height == hw // 8

    fd = FoldedWeights(m.decoder_view(), meta, plan=autoencoder_decoder_plan(m._decoder_config()))
    lat = hw // 8
    prog, em = _record(fd, n, lat, lat, 4, with_embed=False)
    kinds = collections.Counter(k for k, _ in prog.launches)
    assert kinds == collections.Counter(im2col=1, igemm=DEC_IGEMM, conv_out=1)
    assert (em.out_h, em.out_w) == (hw, hw)
    im = prog.launches[0][1]
    assert im.k_pad == 64 and im.src_channels[0] == 4 and im.height == lat
    ds = prog.igemm()
    assert ds[0].c_out == 256 and ds[0].height == lat
    slabs = [d for d in ds if d.n_seg == 2]
    assert len(slabs) == DEC_K_SLABS
    assert [(d.a_channels[0], d.a_taps[0], d.a_channels[1], d.a_taps[1]) for d in slabs] == \
        [(128, 9, 256, 1), (64, 9, 128, 1)]
    assert all(d.epi_flags == 0 for d in slabs)
    assert ds[-1].height == hw and prog.launches[-1][1].c_out == 1 and prog.launches[-1][1].height == hw


def test_decoder_conv_folds_to_the_centre_tap():
    """The 1x1 decoder_conv is folded with its own fan-in and placed on the centre tap (k = 4 * ci + c)."""
    from terrain_diffusion_b200.models.plan import effective_weight
    m = EDMAutoencoder(**CFG).eval()
    m.load_state_dict(oae.procedural_state_dict(CFG, seed=0))
    fd = FoldedWeights(m.decoder_view(), torch.device("cpu"), plan=autoencoder_decoder_plan(m._decoder_config()))
    w_mat = fd.segs["conv_in.im2col"][0][:, :, 0, 0]                     # [256][64]
    w = effective_weight(m.decoder_conv.weight)[:, :, 0, 0]               # [256][5]
    assert torch.equal(w_mat[:, 4 * 5:5 * 5], w)
    assert torch.count_nonzero(w_mat[:, :20]) == 0 and torch.count_nonzero(w_mat[:, 25:]) == 0


def test_im2col_validates_one_and_four_input_channels():
    """1 + ones (encoder) and 4 + ones (decoder) pass the channel check: a wrong k_pad is what is refused."""
    lib = L.lib()
    d = L.TdxIm2colDesc()
    d.src[0], d.out = 16, 16
    d.n_img, d.height, d.width = 1, 8, 8
    for ch in (1, 4):
        d.src_channels[0] = ch
        d.k_pad = 128                           # 9 * 2 = 18 and 9 * 5 = 45 -> must be 64
        assert lib.tdx_im2col_run(C.byref(d), None) != 0
        err = lib.tdx_last_error()
        assert b"k_pad" in err and b"input channels" not in err
    d.src_channels[0] = 2                       # 2 + ones = 3: still refused
    d.k_pad = 64
    assert lib.tdx_im2col_run(C.byref(d), None) != 0 and b"input channels" in lib.tdx_last_error()


def test_bench_autoencoder_help():
    res = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_autoencoder.py"), "--help"], capture_output=True,
                         text=True, timeout=120)
    assert res.returncode == 0 and "--steps" in res.stdout


def test_bench_autoencoder_flop_count():
    sys.path.insert(0, str(ROOT / "tools"))
    try:
        from bench_autoencoder import conv_gflop
    finally:
        sys.path.remove(str(ROOT / "tools"))
    g = conv_gflop(CFG)
    # level 0 alone: four 64->64 3x3 convs at 512^2 in the encoder
    assert g["encode"] > 4 * 2 * 64 * 64 * 9 * 512 * 512 / 1e9
    assert 250 < g["encode"] < 300 and 750 < g["decode"] < 850
