"""The shade kernel's contract (tests/_relief_contract.py), CPU side: held to the device's rule against the oracle
(oracle/relief.py) on every golden case and on the benchmark field of tools/bench_relief.py, so the restatement the GPU
tests compare the kernel with bit for bit is itself shown to agree with the reference; plus its building blocks
(np.gradient written out, the fp32-midpoint test, the statistics buffer) and what the newer golden cases reach."""
from pathlib import Path

import numpy as np
import pytest

from oracle import relief as O
from tests import _relief_contract as K
from tests._relief_inputs import CASES, bench_field, golden_stride, relief_case

G = np.load(Path(__file__).resolve().parent / "golden" / "relief_golden.npz")


def oracle_parts(elev, **kw):
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return O.relief_parts(elev, **kw)


@pytest.mark.parametrize("name", list(CASES))
def test_contract_meets_the_rule_on_golden_cases(name):
    elev, kw = relief_case(name)
    c = K.relief_contract(elev, **kw)
    parts = oracle_parts(elev, **kw)
    n_full, share_full = K.compare(c["rgb"], parts["rgb"], parts)
    s = golden_stride(name)
    n_gold, share_gold = K.compare(c["rgb"][::s, ::s], G[name], {k: v[::s, ::s] for k, v in parts.items()})
    print(f"\ncontract {name}: {K.excuse_summary(c)}; vs oracle {n_full} LUT-boundary px, worst share {share_full:.3f}; "
          f"vs golden {n_gold}, {share_gold:.3f}")


@pytest.mark.parametrize("n", [512, 1024])
def test_contract_meets_the_rule_on_the_benchmark_field(n):
    elev = bench_field(n)
    c = K.relief_contract(elev)
    parts = oracle_parts(elev)
    n_boundary, share = K.compare(c["rgb"], parts["rgb"], parts)
    d, where, on_boundary = K.worst_pixel(c["rgb"], parts["rgb"], parts)
    print(f"\ncontract, benchmark field {n}^2: {K.excuse_summary(c)}; {n_boundary} LUT-boundary px, worst share "
          f"{share:.3f}; worst |diff| {d:.3g} at {where}, {'on' if on_boundary else 'off'} a colormap boundary")
    assert d <= K.TOL or on_boundary


def test_gradient_is_numpys():
    rng = np.random.RandomState(3)
    for shape in ((2, 2), (2, 9), (9, 2), (17, 31)):
        p = (rng.randn(*shape) * 300).astype(np.float32)
        dy, dx = K.gradient(p)
        gy, gx = np.gradient(p)
        assert gy.dtype == np.float32
        assert np.array_equal(dy.view(np.uint32), gy.view(np.uint32)), shape
        assert np.array_equal(dx.view(np.uint32), gx.view(np.uint32)), shape


def test_near_f32_midpoint():
    one = np.float64(1.0)
    mid = one + 2.0 ** -24                                 # halfway between 1 and the next fp32
    ulp = np.spacing(mid)
    assert K.near_f32_midpoint(np.array([mid, mid + 8 * ulp, mid - 8 * ulp]), 8 * ulp).all()
    assert not K.near_f32_midpoint(np.array([mid + 9 * ulp, one, np.nan, np.inf]), 8 * ulp).any()
    below = one - 2.0 ** -25                              # halfway between 1 and the fp32 below it
    assert K.near_f32_midpoint(np.array([below]), 0.0).all()


def test_stats_buffer_encoding():
    x = np.array([5.0, -0.0, np.nan, 3.0, -np.inf, np.nan], np.float32)
    s = K.encode_stats(x)
    assert s[0] == 2
    lo, hi = K.decode_stats(s)
    assert np.array([lo], np.float32).view(np.uint32)[0] == 0 and hi == 5.0     # -0 and -inf count as +0
    assert K.decode_range(s, 0, 0, 0, 0) == (np.float32(0), np.float32(5.0 + 1e-8), True)
    allnan = K.encode_stats(np.full(4, np.nan, np.float32))
    assert allnan[0] == 4 and K.is_fallback(*K.decode_stats(allnan))
    assert K.decode_range(allnan, 0, 0, 0, 0) == (np.float32(0), np.float32(1.0 + 1e-8), True)
    assert K.is_fallback(*K.decode_stats(K.encode_stats(np.array([2.0, np.inf], np.float32))))
    assert K.is_fallback(*K.decode_stats(K.encode_stats(np.full(3, 7.5, np.float32))))
    assert K.decode_range(s, 1, 300.0, 1500.5, 0) == (np.float32(300.0), np.float32(1500.5), False)


def test_newer_golden_cases_reach_their_branches():
    elev, kw = relief_case("inf")
    assert np.isposinf(elev).any() and np.isneginf(elev).any()
    assert K.is_fallback(*K.decode_stats(K.encode_stats(elev))) and np.isnan(G["inf"]).any()
    elev, kw = relief_case("relief2")
    c = K.relief_contract(elev, **kw)
    assert kw["relief"] > 1 and (c["gain"] < 0).any() and (G["relief2"] == 0).all(axis=-1).any()
    for name in ("vmin_only", "vmax_only"):                # one bound alone is ignored: the data's range is used
        elev, kw = relief_case(name)
        data = K.relief_contract(elev)
        assert len(kw) == 1 and np.array_equal(K.relief_contract(elev, **kw)["rgb"], data["rgb"])
    elev, kw = relief_case("vmin_above")
    assert kw["vmin"] > np.nanmax(elev) and np.all(G["vmin_above"][elev > 0] == 0)
    elev, _ = relief_case("abyss")
    assert (elev < -10000).any() and (elev > -10000).any()
