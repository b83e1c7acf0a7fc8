"""The evaluation drivers' terrain decode on the GPU: the batched read-out tdx_eval_terrain bit for bit against the
single-plane chain of inference/postproc.py, decode_latents_to_terrain against the reference's own
`_decode_latents_to_terrain` (tests/golden/eval_terrain_golden.npz) under DESIGN section 2 and against
sample_decoder_consistency_tiled followed by the single-plane read-out, and the generator it draws from.

This module also registers tdx_eval_terrain's fenced cases with tests/test_input_extents_gpu.py (and so with
tests/test_pdl_order_gpu.py, which interposes a running kernel in front of every such case) and its fenced arguments in
tests/_fence.FENCED_ARGS.  It is collected before both, and imports without a GPU, so the coverage checks of a CPU-only
run (tests/test_input_extents_cpu.py) see the entry too.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import unet as ounet  # noqa: E402
from terrain_diffusion_b200 import _lib as L  # noqa: E402
from terrain_diffusion_b200.inference import decode_latents_to_terrain, sample_decoder_consistency_tiled  # noqa: E402
from terrain_diffusion_b200.inference import postproc as P  # noqa: E402
from terrain_diffusion_b200.inference.evaluation import eval_terrain  # noqa: E402
from terrain_diffusion_b200.models import EDMUnet2D  # noqa: E402
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler  # noqa: E402
from tests import test_input_extents_gpu as IE  # noqa: E402
from tests._fence import FENCED_ARGS  # noqa: E402
from tests.test_eval_terrain_cpu import CASES, G, Stats, Wrapped, case_inputs, rel_rms  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
RESIDUAL_MEAN, RESIDUAL_STD = 0.3, 1.7        # neither is an fp32 value: both round on the way in, as torch rounds them


def scratch_elems(n, h, w):
    return 2 * n * (8 * h + 16) * (8 * w + 16)


# ------------------------------------------------------------------------------------------------ fenced inputs
FENCED_ARGS["tdx_eval_terrain"] = ("residual", "lowfreq")


@IE.case("tdx_eval_terrain", (1, 1, 1, 0, 0), (2, 5, 7, 0, 1), (3, 1, 9, 0, 0), (1, 8, 8, 1, 1), (2, 6, 9, 1, 0),
         (2, 8, 16, 1, 1), (1, 64, 64, 1, 0))
def _eval_terrain_case(env, n, h, w, denoise, sq):
    H, W = 8 * h, 8 * w
    res = env.inp("residual", IE._rand(60 + n, n, H, W, lo=-2.0, hi=2.0))
    low = env.inp("lowfreq", IE._rand(61 + n, n, h, w, lo=-1.0, hi=2.0))
    out = env.out("out", (n, H, W))
    ns = scratch_elems(n, h, w)
    scratch = env.out("scratch", (ns,), compare=False)
    IE.call("tdx_eval_terrain", res.data_ptr(), low.data_ptr(), n, h, w, RESIDUAL_MEAN, RESIDUAL_STD, P.LOWFREQ_MEAN,
            P.LOWFREQ_STD, denoise, sq, out.data_ptr(), scratch.data_ptr(), ns)


# ------------------------------------------------------------------------------------------------ the read-out
def per_plane(residual, lowfreq, denoise, signed_square):
    """Today's single-plane chain, one image at a time, with the de-normalisation as torch computes it."""
    out = []
    for r, lo in zip(residual, lowfreq):
        r = r * RESIDUAL_STD + RESIDUAL_MEAN
        lo = lo * P.LOWFREQ_STD + P.LOWFREQ_MEAN
        if denoise:
            r, lo = P.laplacian_denoise(r, lo, 5)
        out.append(P._combine(r, P.resize_extrapolated(lo, r.shape), signed_square=signed_square))
    return torch.stack(out)


def planes(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, 8 * h, 8 * w, generator=g).to(DEV), (torch.randn(n, h, w, generator=g) + 0.5).to(DEV))


@pytest.mark.parametrize("n", [1, 3, 10])
@pytest.mark.parametrize("hw", [(8, 8), (64, 64), (8, 16)], ids=["64x64", "512x512", "64x128"])
@pytest.mark.parametrize("denoise", [False, True], ids=["plain", "denoise"])
@pytest.mark.parametrize("sq", [False, True], ids=["sqrt", "squared"])
def test_batched_readout_is_bit_identical_to_the_per_plane_chain(n, hw, denoise, sq):
    res, low = planes(n, *hw, seed=n * 100 + hw[1])
    got = eval_terrain(res, low, RESIDUAL_MEAN, RESIDUAL_STD, denoise, sq)
    want = per_plane(res, low, denoise, sq)
    assert got.shape == want.shape == (n, 8 * hw[0], 8 * hw[1])
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert float(want.std()) > 1.0


def test_readout_argument_errors():
    res, low = planes(2, 8, 8, seed=1)
    out = torch.empty_like(res)
    ns = scratch_elems(2, 8, 8)
    scratch = torch.empty(ns, device=DEV)
    fn = L.lib().tdx_eval_terrain

    def call(*over, **kw):
        args = dict(residual=res.data_ptr(), lowfreq=low.data_ptr(), n=2, h=8, w=8, denoise=1, out=out.data_ptr(),
                     scratch=scratch.data_ptr(), elems=ns)
        args.update(kw)
        L.call(fn, DEV, args["residual"], args["lowfreq"], args["n"], args["h"], args["w"], 0.0, 1.0, 0.0, 1.0,
               args["denoise"], 0, args["out"], args["scratch"], args["elems"])

    call()
    for kw, msg in ((dict(residual=None), "null"), (dict(n=0), "batch"), (dict(h=0), "shape"),
                    (dict(elems=ns - 1), "scratch holds"), (dict(out=res.data_ptr()), "overlap"),
                    (dict(scratch=out.data_ptr()), "overlap"), (dict(h=1, w=1, elems=10 ** 6), "reflect padding"),
                    (dict(h=1, w=9, elems=10 ** 6), "wider than high")):
        with pytest.raises(L.TdxError, match=msg):
            call(**kw)
    with pytest.raises(L.TdxError, match="CPU path"):
        eval_terrain(res.cpu(), low.cpu(), 0.0, 1.0)
    with pytest.raises(ValueError, match="needs"):
        eval_terrain(res[:, :8], low, 0.0, 1.0)


# ------------------------------------------------------------------------------------------------ the decode
@pytest.fixture(scope="module")
def decoder():
    m = EDMUnet2D(**ounet.DECODER_CFG).eval()
    m.load_state_dict(ounet.procedural_state_dict(ounet.DECODER_CFG, seed=0))
    return m.to(DEV)


def decode(case, decoder, **kw):
    samples, noise, inter_t, denoise = case_inputs(case)
    ds = Wrapped(Stats()) if bool(G[f"{case}.wrapped"]) else Stats()
    return decode_latents_to_terrain(samples.to(DEV), ds, decoder, EDMDPMSolverMultistepScheduler(), None, inter_t,
                                     not denoise, noise=noise.to(DEV), **kw)


def assert_meets_golden(case, y):
    want = torch.from_numpy(G[f"{case}.y"])
    err = rel_rms(y.cpu(), want)
    ref = float(G[f"{case}.ref_bf16_err"])
    assert y.shape == want.shape and y.dtype == torch.float32 and y.is_cuda
    assert err <= 1e-2 and err <= 1.25 * ref, f"{case}: rel-RMS {err:.3g}, reference bf16 {ref:.3g}"


@pytest.mark.parametrize("case", CASES)
def test_decode_meets_the_reference(case, decoder):
    assert_meets_golden(case, decode(case, decoder))


@pytest.mark.parametrize("batch", [1, 4, None])
def test_decoder_batch_size_meets_the_reference_and_repeats_bit_for_bit(batch, decoder):
    y = decode("a", decoder, decoder_batch_size=batch)
    assert_meets_golden("a", y)
    assert torch.equal(decode("a", decoder, decoder_batch_size=batch).view(torch.int32), y.view(torch.int32))


@pytest.mark.parametrize("case", CASES)
def test_decode_matches_the_tiled_sampler_and_the_per_plane_readout(case, decoder):
    samples, noise, inter_t, denoise = case_inputs(case)
    st = Stats()
    samples, noise = samples.to(DEV), noise.to(DEV)
    B, _, h, w = samples.shape
    cond = torch.nn.functional.interpolate(samples[:, :4] / st.latents_std.to(DEV) + st.latents_mean.to(DEV),
                                           size=(8 * h, 8 * w), mode="nearest")
    residual = sample_decoder_consistency_tiled(decoder, EDMDPMSolverMultistepScheduler(), cond, noise, 8 * h, 8 * h,
                                                intermediate_t=inter_t)
    want = []
    for r, lo in zip(residual[:, 0], samples[:, 4]):
        r = r * st.residual_std + st.residual_mean
        lo = lo * P.LOWFREQ_STD + P.LOWFREQ_MEAN
        if denoise:
            r, lo = P.laplacian_denoise(r, lo, 5)
        want.append(P.laplacian_decode(r, lo, extrapolate=True))
    want = torch.stack(want)[:, None]
    assert rel_rms(decode(case, decoder), want) <= 2e-3


def test_one_draw_from_the_generator_as_the_reference_draws(decoder):
    samples, _, inter_t, denoise = case_inputs("b")
    B, _, h, w = samples.shape
    g = torch.Generator(device=DEV).manual_seed(77)
    ref = torch.Generator(device=DEV).manual_seed(77)
    z = torch.randn((B, 1, 8 * h, 8 * w), generator=ref, device=DEV, dtype=torch.float32)
    y = decode_latents_to_terrain(samples.to(DEV), Stats(), decoder, EDMDPMSolverMultistepScheduler(), g, inter_t,
                                  not denoise)
    assert torch.equal(g.get_state(), ref.get_state())
    y_explicit = decode_latents_to_terrain(samples.to(DEV), Stats(), decoder, EDMDPMSolverMultistepScheduler(), None,
                                           inter_t, not denoise, noise=z)
    assert torch.equal(y.view(torch.int32), y_explicit.view(torch.int32))


def test_signed_square_is_the_square_of_the_terrain(decoder):
    y = decode("b", decoder)
    y2 = decode("b", decoder, signed_square=True)
    assert torch.equal(y2, torch.sign(y) * y * y)
