"""The decoder evaluations on the GPU: the batched pre-padded read-out tdx_eval_padded_terrain bit for bit against the
single-plane chain of inference/postproc.py and within DESIGN section 4.4 of the reference's own laplacian_decode, and
decoder_eval_terrain against the reference's drivers (tests/golden/decoder_eval_golden.npz) under DESIGN section 2, across
tile batches, on repeat, and for the generator it draws from.

This module also registers tdx_eval_padded_terrain's fenced cases with tests/test_input_extents_gpu.py (and so with
tests/test_pdl_order_gpu.py, which interposes a running kernel in front of every such case) and its fenced arguments in
tests/_fence.FENCED_ARGS.  It is collected before both, and imports without a GPU, so the coverage checks of a CPU-only
run (tests/test_input_extents_cpu.py) see the entry too.
"""
from __future__ import annotations

import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import unet as ounet  # noqa: E402
from terrain_diffusion_b200 import _lib as L  # noqa: E402
from terrain_diffusion_b200.inference import decoder_eval_terrain, normalize_uint8_three_channel  # noqa: E402
from terrain_diffusion_b200.inference import padded_terrain  # noqa: E402
from terrain_diffusion_b200.inference import postproc as P  # noqa: E402
from terrain_diffusion_b200.models import EDMUnet2D  # noqa: E402
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler  # noqa: E402
from tests import _decoder_eval_inputs as I  # noqa: E402
from tests import test_input_extents_gpu as IE  # noqa: E402
from tests._fence import FENCED_ARGS  # noqa: E402
from tests.test_decoder_eval_cpu import G, rel_rms, sub  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
RESIDUAL_MEAN, RESIDUAL_STD = 0.3, 1.7        # neither is an fp32 value: both round on the way in, as torch rounds them


def scratch_elems(n, h, w):
    return n * (h + 2) * (8 * w + 16)


# ------------------------------------------------------------------------------------------------ fenced inputs
FENCED_ARGS["tdx_eval_padded_terrain"] = ("residual", "lowfreq_padded")


@IE.case("tdx_eval_padded_terrain", (1, 1, 1, 0, 0), (2, 5, 7, 1, 0), (3, 1, 9, 0, 8), (1, 8, 8, 1, 64),
         (2, 6, 9, 1, 17), (2, 16, 16, 0, 0))
def _eval_padded_terrain_case(env, n, h, w, sq, crop):
    H, W = 8 * h, 8 * w
    c = crop or None
    res = env.inp("residual", IE._rand(70 + n, n, H, W, lo=-2.0, hi=2.0))
    low = env.inp("lowfreq_padded", IE._rand(71 + n, n, h + 2, w + 2, lo=-1.0, hi=30.0))
    out = env.out("out", (n, c or H, c or W))
    ns = scratch_elems(n, h, w)
    scratch = env.out("scratch", (ns,), compare=False)
    IE.call("tdx_eval_padded_terrain", res.data_ptr(), low.data_ptr(), n, h, w, RESIDUAL_MEAN, RESIDUAL_STD, sq, crop,
            out.data_ptr(), scratch.data_ptr(), ns)


# ------------------------------------------------------------------------------------------------ the read-out
def per_plane(residual, lowfreq_padded, signed_square, crop=None, mean=RESIDUAL_MEAN, std=RESIDUAL_STD):
    """Today's single-plane chain, one plane at a time, with the de-normalisation as torch computes it:
    laplacian_decode(pre_padded=True) is the resize to (H + 16) x (W + 16), the crop by 8, then the combine."""
    out = []
    for r, lo in zip(residual, lowfreq_padded):
        H, W = r.shape
        up = P.resize_bilinear(lo, (H + 16, W + 16))[8:8 + H, 8:8 + W]
        t = P._combine(r * std + mean, up, signed_square=signed_square)
        if crop:
            i, j = (H - crop) // 2, (W - crop) // 2
            t = t[i:i + crop, j:j + crop]
        out.append(t)
    return torch.stack(out)


def planes(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, 8 * h, 8 * w, generator=g).to(DEV),
            (torch.randn(n, h + 2, w + 2, generator=g) * 8 + 20).to(DEV))


@pytest.mark.parametrize("n", [1, 3, 20])
@pytest.mark.parametrize("hw, crop", [((8, 8), None), ((64, 64), None), ((112, 112), 512)],
                         ids=["64x64", "512x512", "896x896-crop512"])
@pytest.mark.parametrize("sq", [False, True], ids=["plain", "squared"])
def test_batched_readout_is_bit_identical_to_the_per_plane_chain(n, hw, crop, sq):
    res, low = planes(n, *hw, seed=n * 100 + hw[1])
    got = padded_terrain(res, low, RESIDUAL_MEAN, RESIDUAL_STD, sq, crop)
    want = per_plane(res, low, sq, crop)
    side = crop or 8 * hw[0]
    assert got.shape == want.shape == (n, side, side)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert float(want.std()) > 1.0


def test_readout_argument_errors():
    res, low = planes(2, 8, 8, seed=1)
    out = torch.empty_like(res)
    ns = scratch_elems(2, 8, 8)
    scratch = torch.empty(ns, device=DEV)
    fn = L.lib().tdx_eval_padded_terrain

    def call(**kw):
        args = dict(residual=res.data_ptr(), lowfreq=low.data_ptr(), n=2, h=8, w=8, crop=0, out=out.data_ptr(),
                    scratch=scratch.data_ptr(), elems=ns)
        args.update(kw)
        L.call(fn, DEV, args["residual"], args["lowfreq"], args["n"], args["h"], args["w"], 0.0, 1.0, 1, args["crop"],
               args["out"], args["scratch"], args["elems"])

    call()
    for kw, msg in ((dict(residual=None), "null"), (dict(n=0), "batch"), (dict(h=0), "shape"),
                    (dict(crop=65), "crop"), (dict(crop=-1), "crop"), (dict(elems=ns - 1), "scratch holds"),
                    (dict(out=res.data_ptr()), "overlap"), (dict(scratch=out.data_ptr()), "overlap"),
                    (dict(out=low.data_ptr(), crop=4), "overlap")):
        with pytest.raises(L.TdxError, match=msg):
            call(**kw)
    for r, lo in ((res[:, :8], low), (res, low[:, :9]), (res[:, :, :60], low), (res[:, :16, :16], low[:, :3, :3])):
        with pytest.raises(ValueError, match="takes"):
            padded_terrain(r, lo, 0.0, 1.0)
    with pytest.raises(ValueError, match="crop"):
        padded_terrain(res, low, 0.0, 1.0, crop=65)


def _golden_batches():
    for case in I.CASES:
        for k, batch in enumerate(I.batches(case)):
            yield case, k, batch


def assert_readout_close(got, want, what):
    """The read-out against the reference's torchvision CPU resize, which rounds its fused multiply-adds differently:
    within DESIGN section 4.4's bound, 1e-5 of the plane's largest magnitude."""
    err = float((got.cpu() - want).abs().max())
    assert err <= 1e-5 * float(want.abs().max()), f"{what}: max |diff| {err:.3g} of {float(want.abs().max()):.3g}"


def test_readout_matches_the_references_laplacian_decode():
    """Every real image of the golden runs (read out from images / sigma_data, as the drivers do) and the generated
    images of case dc (from the de-normalised argument the reference's laplacian_decode received)."""
    n_fake = 0
    for case in I.CASES:
        for k, batch in enumerate(I.batches(case)):
            images, lp = batch["image"].to(DEV), batch["lowfreq_padded"][:, 0].to(DEV)
            real = padded_terrain((images / I.SIGMA_DATA)[:, 0], lp, I.RESIDUAL_MEAN, I.RESIDUAL_STD, True,
                                  I.CASES[case]["crop"])
            assert_readout_close(sub(real[:, None], case), torch.from_numpy(G[f"{case}.{k}.real"]), (case, k))
            if f"{case}.{k}.fake_ld_arg" in G:
                arg = torch.from_numpy(G[f"{case}.{k}.fake_ld_arg"]).to(DEV)[:, 0]
                fake = padded_terrain(arg, lp, 0.0, 1.0, False)
                assert_readout_close(sub(fake[:, None], case), torch.from_numpy(G[f"{case}.{k}.fake_ld"]), (case, k))
                n_fake += 1
    assert n_fake == 1


# ------------------------------------------------------------------------------------------------ the decode
@pytest.fixture(scope="module")
def decoder():
    m = EDMUnet2D(**ounet.DECODER_CFG).eval()
    m.load_state_dict(ounet.procedural_state_dict(ounet.DECODER_CFG, seed=0))
    return m.to(DEV)


def run(case, decoder, batch, generator, **kw):
    c = I.CASES[case]
    return decoder_eval_terrain(decoder, EDMDPMSolverMultistepScheduler(), batch["image"].to(DEV),
                                batch["lowfreq_padded"].to(DEV), batch["cond_img"].to(DEV), generator,
                                residual_mean=I.RESIDUAL_MEAN, residual_std=I.RESIDUAL_STD, sigma_data=I.SIGMA_DATA,
                                tile_size=c["tile_size"], tile_stride=c["tile_stride"],
                                intermediate_sigma=c["intermediate_sigma"], crop_size=c["crop"], **kw)


@pytest.mark.parametrize("case", tuple(I.CASES))
def test_decoder_eval_meets_the_reference(case, decoder):
    """The driver loop with decoder_eval_terrain and normalize_uint8_three_channel swapped in, fed the golden's
    batches and the drivers' CPU generator: the generated terrain within DESIGN section 2 of the reference's, the real
    terrain within the read-out's bound and its uint8 image within one level at rounding boundaries, the generated
    uint8 image within one level of the reference's own bf16 difference."""
    g = torch.Generator().manual_seed(I.GENERATOR_SEED)
    fakes, wants = [], []
    for k, batch in enumerate(I.batches(case)):
        fake, real = run(case, decoder, batch, g)
        side = I.CASES[case]["crop"] or I.CASES[case]["size"]
        assert fake.shape == real.shape == (batch["image"].shape[0], 1, side, side)
        assert fake.dtype == torch.float32 and fake.is_cuda
        assert_readout_close(sub(real, case), torch.from_numpy(G[f"{case}.{k}.real"]), (case, k))
        fake_u8, real_u8 = normalize_uint8_three_channel(fake), normalize_uint8_three_channel(real)
        dr = (sub(real_u8, case).cpu().int() - torch.from_numpy(G[f"{case}.{k}.real_u8"]).int()).abs()
        assert int(dr.max()) <= 1 and float(dr.float().mean()) < 1e-3
        du8 = (sub(fake_u8, case).cpu().int() - torch.from_numpy(G[f"{case}.{k}.fake_u8"]).int()).abs()
        assert int(du8.max()) <= max(1, int(G[f"{case}.ref_bf16_u8_diff"])) + 1
        fakes.append(sub(fake, case).cpu())
        wants.append(torch.from_numpy(G[f"{case}.{k}.fake"]))
    assert k + 1 == int(G[f"{case}.batches"])
    err, ref = rel_rms(torch.cat(fakes), torch.cat(wants)), float(G[f"{case}.ref_bf16_err"])
    assert err <= 1e-2 and err <= 1.25 * ref, f"{case}: rel-RMS {err:.3g}, reference bf16 {ref:.3g}"


@pytest.mark.parametrize("case", ("dc", "tiled"))
def test_tile_batches_agree_and_repeat_bit_for_bit(case, decoder):
    batch = next(I.batches(case))
    out = {}
    for tb in (1, None):
        runs = [run(case, decoder, batch, torch.Generator(device=DEV).manual_seed(5), tile_batch=tb) for _ in range(2)]
        for a, b in zip(runs[0], runs[1]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        out[tb] = runs[0]
    assert rel_rms(out[1][0], out[None][0]) <= 2e-3
    assert torch.equal(out[1][1], out[None][1])


@pytest.mark.parametrize("case", ("dc", "dc1"))
def test_draws_from_the_generator_as_the_drivers_draw(case, decoder):
    c = I.CASES[case]
    batch = next(I.batches(case))
    B, T = batch["image"].shape[0], c["tile_size"]
    n_tiles = ((c["size"] - T) // c["tile_stride"] + 1) ** 2
    n_steps = 2 if c["intermediate_sigma"] > 0 else 1
    g = torch.Generator(device=DEV).manual_seed(77)
    ref = torch.Generator(device=DEV).manual_seed(77)
    for _ in range(n_tiles * n_steps):
        torch.randn((B, 1, T, T), generator=ref, device=DEV)
    run(case, decoder, batch, g)
    assert torch.equal(g.get_state(), ref.get_state())
    assert torch.equal(torch.randn(5, generator=g, device=DEV), torch.randn(5, generator=ref, device=DEV))
