"""The overlapped-epilogue implicit-GEMM kernel (cluster-free launches with N <= 128, several items per CTA and no
pixel-norm statistics: a third warpgroup runs the epilogue while the MMA warpgroups go on to the next item) against the
serial-epilogue kernel, bit for bit.

Both kernels issue the same MMAs in the same order and the same epilogue arithmetic in the same order, so every output
byte must agree.  The serial kernel is selected through the debug hook tdx_debug_igemm_serial_epilogue; the launch plan
is the same either way.  Cases: every (plan class, epilogue signature) of the decoder's overlapped 256^2 and 128^2
launches in a one-tile and a 16-tile forward (the bench's shapes); then every other (plan variant, epilogue signature)
group of the shape surface (tests/_igemm_surface.py) that runs on the overlapped kernel; plus hand-written cases for the
epilogue paths and item counts the surface may not reach on a given GPU.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import functools

import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from tests._igemm_ref import Case, make_inputs, plan_class, plan_label, plan_of, report, run_cuda
from tests._igemm_surface import (BENCH_TILE, BENCH_TILES, Forward, epilogue_signature, gpu_tests_selected,
                                  group_key, group_representatives, launches, new_groups)

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


@functools.lru_cache(maxsize=None)
def decoder_cases() -> tuple:
    """The fewest-MAC launch of every (plan class, epilogue signature) among the decoder's overlapped 256^2 and 128^2
    launches at the bench's 1 and 16 tiles."""
    groups: dict = {}
    for la in launches():
        if la.forward.model != "decoder" or la.forward.hw != BENCH_TILE or la.forward.n not in BENCH_TILES:
            continue
        if la.case.h not in (256, 128) or not la.plan["ov"]:
            continue
        key = (plan_class(la.plan), epilogue_signature(la.case))
        if key not in groups or la.case.macs < groups[key].macs:
            groups[key] = dataclasses.replace(la.case, name=f"decoder_b{la.forward.n}:{la.layer}")
    return tuple(dataclasses.replace(c, name=f"{plan_label(cls)}-{c.name}")
                 for (cls, _), c in sorted(groups.items(), key=lambda kv: str(kv[0])))


@functools.lru_cache(maxsize=None)
def surface_cases() -> tuple:
    """The representative of every surface group on the overlapped kernel that decoder_cases() leaves out."""
    done = {group_key(c, plan_of(c)) for c in decoder_cases()}
    return tuple(c for c in group_representatives() if plan_of(c)["ov"] and group_key(c, plan_of(c)) not in done)


def pytest_generate_tests(metafunc):
    cases = {"test_decoder_plan_overlapped_matches_serial": decoder_cases,
             "test_surface_plan_overlapped_matches_serial": surface_cases}.get(metafunc.function.__name__)
    if cases is not None:
        metafunc.parametrize("case", cases() if gpu_tests_selected(metafunc.config) else (), ids=lambda c: c.name)


@pytest.fixture(scope="module")
def compared() -> set:
    """Names of the cases found bit-identical to the serial kernel in this session."""
    return set()


def _serial(on: bool) -> None:
    fn = L.lib().tdx_debug_igemm_serial_epilogue
    fn.restype = None
    fn.argtypes = [C.c_int32]
    fn(1 if on else 0)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def check_bit_identical(case: Case) -> None:
    assert plan_of(case)["ov"], f"{case.name}: plan {plan_of(case)} does not run the overlapped kernel"
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


def test_decoder_plan_overlapped_matches_serial(case, compared):
    check_bit_identical(case)
    compared.add(case.name)


def test_surface_plan_overlapped_matches_serial(case, compared):
    check_bit_identical(case)
    compared.add(case.name)


@pytest.mark.parametrize("case", HAND_CASES, ids=lambda c: c.name)
def test_hand_case_overlapped_matches_serial(case):
    check_bit_identical(case)


def test_cases_cover_the_epilogue_paths(request, compared):
    """Every surface group on the overlapped kernel is compared with the serial kernel by one of the two parametrized
    tests above (or here, if they have not compared it in this session), and between them the cases reach several
    rounds per CTA with a partial last round, both N, and every epilogue feature the overlapped kernel takes.  Writes
    the number of overlapped groups, and of those no PRODUCT forward reaches, to the terminal (also under -q)."""
    assert decoder_cases(), "no overlapped 256^2 / 128^2 launch in the decoder forward"
    ov = list(decoder_cases()) + list(surface_cases())
    keys = {group_key(la.case, la.plan) for la in launches() if la.plan["ov"]}
    compared_keys = {group_key(c, plan_of(c)) for c in ov}
    assert keys <= compared_keys, sorted(map(str, keys - compared_keys))
    for c in ov:
        if c.name not in compared:
            check_bit_identical(c)
    new = new_groups()
    report(request.config, [f"igemm overlapped kernel: {len(keys)} surface groups ({len(ov)} cases) bit-identical to "
                            f"the serial kernel, {sum(1 for k in keys if k in new)} of them reached by no PRODUCT "
                            f"forward; {len(HAND_CASES)} hand-written cases"])
    cases = ov + HAND_CASES
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
