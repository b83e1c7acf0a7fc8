"""The overlapped-epilogue implicit-GEMM kernel (cluster-free launches with N <= 128, several items per CTA and no
pixel-norm statistics: a third warpgroup runs the epilogue while the MMA warpgroups go on to the next item) against the
serial-epilogue kernel, bit for bit.

Both kernels issue the same MMAs in the same order and the same epilogue arithmetic in the same order, so every output
byte must agree.  The serial kernel is selected through the debug hook tdx_debug_igemm_serial_epilogue; the launch plan
is the same either way.  Cases: every (plan class, epilogue signature) of the decoder's 256^2 and 128^2 launches in a
one-tile and a 16-tile forward (the bench's shapes), plus hand-written cases for the epilogue paths and item counts
those forwards may not reach on a given GPU.
"""
from __future__ import annotations

import ctypes as C
import functools

import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from tests._capture import capture_forward, layer_of
from tests._igemm_ref import Case, case_from_desc, make_inputs, needs_norm, plan_class, plan_label, plan_of, run_cuda

pytestmark = pytest.mark.gpu

E, R = L.EPI_EMB_SILU, L.EPI_RESID
RAW, SILU = L.OUT_RAW, L.OUT_SILU
SAME, UP2, DOWN2 = L.SP_SAME, L.SP_UP2, L.SP_DOWN2

HAND_CASES = [
    # residual with its pixel-norm from the producer's side plane, clip, raw + down2 + up2 outputs, about four rounds
    # per CTA with a partial last round
    Case("ov_n64_resid_inv_3outs", [(64, 9)], 64, 4, 128, 128, epi=R, resid_pnorm=1, resid_inv=True, clip=256.0,
         outs=[(RAW, SAME, 1.0), (SILU, DOWN2, 1.0), (SILU, UP2, 0.8)]),
    # residual with its pixel-norm recomputed (all Cout channels read per pixel: two partial sums), double-resolution
    # residual
    Case("ov_n64_resid_pnorm_double_res", [(64, 9)], 64, 2, 128, 128, epi=R, resid_spatial=DOWN2, resid_pnorm=1,
         outs=[(RAW, SAME, 1.0), (SILU, SAME, 1.0)]),
    # the same over 128 channels, N = 128 (four chunks per epilogue thread)
    Case("ov_n128_resid_pnorm_up2", [(128, 9)], 128, 2, 128, 128, epi=R, resid_pnorm=1, n_item=128,
         outs=[(RAW, SAME, 1.0), (SILU, UP2, 1.0)]),
    # residual without pixel-norm, N = 128, three segments
    Case("ov_n128_resid_3seg", [(128, 9), (64, 1), (64, 1)], 128, 2, 128, 128, epi=R, resid_scale=0.9, n_item=128,
         outs=[(RAW, SAME, 1.0), (SILU, SAME, 1.1)]),
    # emb-silu on many rounds, weights streamed (N = 128 items over 128 output channels of 256 inputs)
    Case("ov_n128_emb_stream", [(256, 9)], 128, 8, 64, 64, epi=E, n_item=128),
    # ragged image: the last tile row is half outside, several images
    Case("ov_n64_ragged_emb", [(64, 9)], 64, 3, 136, 120, epi=E),
    # two channel slices of one M tile without pixel-norm stay cluster-free
    Case("ov_n64_two_slices_resid_half_res", [(64, 9)], 128, 2, 128, 128, epi=R, resid_spatial=UP2, n_item=64,
         outs=[(RAW, SAME, 1.0), (SILU, SAME, 1.2)]),
]


def overlapped(case: Case, plan: dict) -> bool:
    """Whether igemm_launch runs this launch on the overlapped kernel."""
    return plan["cluster"] == 1 and plan["N"] <= 128 and plan["rounds"] > 1 and not needs_norm(case)


def epilogue_signature(c: Case) -> tuple:
    return (c.epi, c.resid_spatial if c.epi & R else None, c.resid_pnorm, c.resid_inv, c.rms_out,
            tuple((k, s) for k, s, _ in c.outs), c.clip > 0, tuple(t for _, t in c.segs))


@functools.lru_cache(maxsize=None)
def decoder_cases() -> tuple:
    """The fewest-MAC launch of every (plan class, epilogue signature) among the decoder's overlapped 256^2 and 128^2
    launches at batch 1 and 16."""
    groups: dict = {}
    for n in (1, 16):
        prog = capture_forward("decoder", n, 256)
        for d in prog.igemm():
            if d.height not in (256, 128):
                continue
            c = case_from_desc(d, name=f"decoder_b{n}:{layer_of(prog, d)}")
            p = plan_of(c)
            if not overlapped(c, p):
                continue
            key = (plan_class(p), epilogue_signature(c))
            if key not in groups or c.macs < groups[key].macs:
                groups[key] = c
    cases = []
    for (cls, _), c in sorted(groups.items(), key=lambda kv: str(kv[0])):
        c.name = f"{plan_label(cls)}-{c.name}"
        cases.append(c)
    return tuple(cases)


def pytest_generate_tests(metafunc):
    if metafunc.function.__name__ == "test_decoder_plan_overlapped_matches_serial":
        cases = decoder_cases() if torch.cuda.is_available() else ()
        metafunc.parametrize("case", cases, ids=lambda c: c.name)


def _serial(on: bool) -> None:
    fn = L.lib().tdx_debug_igemm_serial_epilogue
    fn.restype = None
    fn.argtypes = [C.c_int32]
    fn(1 if on else 0)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def check_bit_identical(case: Case) -> None:
    assert overlapped(case, plan_of(case)), f"{case.name}: plan {plan_of(case)} does not run the overlapped kernel"
    inputs = make_inputs(case, "cuda:0")
    try:
        _serial(True)
        ref = run_cuda(case, *inputs)
    finally:
        _serial(False)
    got = run_cuda(case, *inputs)
    assert len(got) == len(ref)
    for i, (g, r) in enumerate(zip(got, ref)):
        what = "rms_out" if i == len(case.outs) else f"out{i}"
        assert not torch.isnan(r.float()).any(), f"{case.name} {what}: the serial kernel left elements unwritten"
        diff = int((_bits(g) != _bits(r)).sum())
        assert diff == 0, f"{case.name} {what}: {diff} elements differ from the serial-epilogue kernel"


def test_decoder_plan_overlapped_matches_serial(case):
    check_bit_identical(case)


@pytest.mark.parametrize("case", HAND_CASES, ids=lambda c: c.name)
def test_hand_case_overlapped_matches_serial(case):
    check_bit_identical(case)


def test_cases_cover_the_epilogue_paths():
    """Between them the cases reach several rounds per CTA with a partial last round, both N, and every epilogue
    feature the overlapped kernel takes."""
    cases = list(decoder_cases()) + HAND_CASES
    assert decoder_cases(), "no overlapped 256^2 / 128^2 launch in the decoder forward"
    plans = [plan_of(c) for c in cases]
    features = {
        "several rounds, partial last": any(p["rounds"] >= 3 and p["partial"] for p in plans),
        "N = 64": any(p["N"] == 64 for p in plans),
        "N = 128": any(p["N"] == 128 for p in plans),
        "emb-silu": any(c.epi & E for c in cases),
        "residual, pixel-norm recomputed": any(c.epi & R and c.resid_pnorm and not c.resid_inv for c in cases),
        "residual, resid_inv plane": any(c.epi & R and c.resid_inv for c in cases),
        "residual, no pixel-norm": any(c.epi & R and not c.resid_pnorm for c in cases),
        "down2 output": any(s == DOWN2 for c in cases for _, s, _ in c.outs),
        "up2 output": any(s == UP2 for c in cases for _, s, _ in c.outs),
    }
    assert all(features.values()), [k for k, v in features.items() if not v]
