"""River routing, CPU side: the oracle restatement (oracle/hydrology.py) against the golden vectors recorded from the
reference's own d8_flow / flow_accumulation / plot_flow_indicator (tests/golden/make_golden_hydrology.py), the
adversarial serpentine input, and the argument checks of terrain_diffusion_b200.inference.hydrology."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import hydrology as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import hydrology as H
from oracle import depressions as OD
from tests._hydrology_inputs import CASES, FILLED_CASES, hydrology_case, serpentine

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "hydrology_golden.npz")


def ulps(a, b) -> int:
    """Largest distance in units in the last place between two fp32 arrays of non-negative values."""
    return int(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)).max(initial=0))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(name):
    z, tol, pools = hydrology_case(name)
    rr, cc, is_sink, kmax = O.d8(z, tol)
    assert np.array_equal(kmax, G[f"{name}.kmax"]) and np.array_equal(is_sink, G[f"{name}.is_sink"])
    a = O.accumulate(z, rr, cc, is_sink)
    assert a.dtype == np.float32 and np.array_equal(a.view(np.uint32), G[f"{name}.A"].view(np.uint32))
    for k in pools:                                          # the indicator routes with the default tol
        got, g = O.flow_indicator(z, k), G[f"{name}.ind{k}"]
        assert got.dtype == np.float32 and got.shape == g.shape
        assert ulps(got, g) <= 1, (k, ulps(got, g))        # numpy's fp32 log1p depends on the host's SIMD path


@pytest.mark.parametrize("name", list(FILLED_CASES))
def test_oracle_routes_the_reference_fill_of_a_neg_inf_dem(name):
    build, pools = FILLED_CASES[name]
    z = build()
    filled = G[f"{name}.filled"]
    assert np.isneginf(z).any() and np.array_equal(np.isneginf(filled), np.isneginf(z))   # the ocean stays -inf
    assert np.array_equal(OD.fill(z)[0].view(np.uint32), filled.view(np.uint32))
    rr, cc, is_sink, kmax = O.d8(filled)
    assert np.array_equal(kmax, G[f"{name}.kmax"]) and np.array_equal(is_sink, G[f"{name}.is_sink"])
    assert np.array_equal(O.accumulate(filled, rr, cc, is_sink).view(np.uint32), G[f"{name}.A"].view(np.uint32))
    for k in pools:
        assert ulps(O.flow_indicator(filled, k), G[f"{name}.ind{k}"]) <= 1


def test_neg_inf_goldens_cover_the_ocean_rules():
    # -inf centres are sinks that route north (kmax 0, the argmax of an all -inf column); land beside -inf prefers it
    for name in ("neg_inf", "neg_inf_seams", "neg_inf_all"):
        z, _, _ = hydrology_case(name)
        ninf = np.isneginf(z)
        assert ninf.any() and np.all(G[f"{name}.is_sink"][ninf]) and np.all(G[f"{name}.kmax"][ninf] == 0)
        assert np.all(G[f"{name}.A"][ninf] == 0)
    z, _, _ = hydrology_case("neg_inf")
    assert np.isneginf(z[[0, 0, -1, -1], [0, -1, 0, -1]]).all()                   # all four corners
    rr, cc, _, _ = O.d8(z)
    beside = ~O.ocean(z) & ~G["neg_inf.is_sink"] & np.isneginf(z[rr, cc])
    assert beside.sum() > 40                                   # land draining into -inf ocean, which is not followed
    assert np.isnan(z[8, 14]) and np.isneginf(z[8, 13])       # NaN beside -inf


def test_golden_cases_cover_the_branches():
    # an exact slope of fp32(tol) is kept: the tol comparison happens in fp32
    z, tol, _ = hydrology_case("tol_between")
    assert np.float32(tol) == np.float32(0.125) and tol > 0.125
    assert not np.array_equal(O.d8(z, np.nextafter(np.float32(0.125), np.float32(1)))[3], G["tol_between.kmax"])
    # plateaus: flat land sinks, and equal best slopes in more than one direction (the k-order tie-break)
    z, _, _ = hydrology_case("plateau")
    assert (G["plateau.is_sink"] & ~O.ocean(z)).sum() > 100 and (z == -0.0).any() and (z == 0.0).any()
    # border ocean read through edge-clamped neighbours; pool results that are empty
    z, _, _ = hydrology_case("edge_ocean")
    interior = O.ocean(z)[1:-1, 1:-1]
    assert O.ocean(z).any() and not interior.any()
    assert G["row.ind2"].shape == (0, 18) and G["two.ind3"].shape == (0, 0) and G["col.ind3"].shape == (9, 0)
    assert np.all(G["all_nan.A"] == 0) and np.all(G["all_ocean.A"] == 0)
    assert float(G["big.A"].max()) > 1000                   # long rivers in the 256^2 case


def test_serpentine_is_one_long_path():
    z, path = serpentine(32)
    rr, cc, is_sink, _ = O.d8(z)
    recv = O.receivers(z, rr, cc, is_sink)
    assert np.array_equal(recv[path[:-1]], path[1:]) and recv[path[-1]] == -1
    assert len(path) == 32 * 32 // 2 + 32 // 2 - 1
    a = O.accumulate(z, rr, cc, is_sink)
    assert a.ravel()[path[-1]] == 32 * 32 and np.all(np.diff(a.ravel()[path]) > 0)


def test_argument_errors_and_positive_inf_come_before_any_device_work(monkeypatch):
    # +inf (and a value that rounds to it in fp32) is refused on the host; -inf is ocean and reaches the device
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(L, "lib", no_device)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    z = np.full((6, 7), 10.0, np.float32)
    idx = np.zeros((6, 7), np.int64)
    sink = np.zeros((6, 7), bool)
    fns = (H.d8_flow, H.plot_flow_indicator, lambda x: H.flow_accumulation(x, idx, idx, sink))
    for bad in (np.zeros(5, np.float32), np.zeros((0, 4), np.float32), np.zeros((3, 0), np.float32),
                np.zeros((2, 3, 4), np.float32), np.zeros((6, 7), np.int32), torch.zeros(6, 7, dtype=torch.int64),
                np.zeros((4097, 4096), np.float32), torch.zeros(1, 2 ** 24 + 1)):
        for fn in fns[:2]:
            with pytest.raises(ValueError):
                fn(bad)
    for bad_value in (np.inf, 1e300):                        # 1e300 is +inf in fp32
        zb = z.astype(np.float64)
        zb[2, 3] = bad_value
        for fn in fns:
            with pytest.raises(ValueError, match=r"\+inf"):
                fn(zb)
        with pytest.raises(ValueError, match=r"\+inf"):
            H.d8_flow(torch.from_numpy(zb))                  # CPU tensor: checked on the host
    for ocean_value in (-np.inf, -1e300):                    # -inf is ocean: it passes the host checks
        zb = z.astype(np.float64)
        zb[2, 3] = ocean_value
        for fn in fns:
            with pytest.raises(L.TdxError):
                fn(zb)
    with pytest.raises(ValueError):
        H.flow_accumulation(z, idx[:5], idx, sink)
    with pytest.raises(ValueError):
        H.flow_accumulation(z, idx, idx, sink[:, :6])
    with pytest.raises(ValueError):
        H.flow_accumulation(z, idx.astype(np.float64), idx, sink)
    with pytest.raises(ValueError):
        H.flow_accumulation(z, idx, torch.zeros(6, 7), sink)
    with pytest.raises(ValueError):
        H.flow_accumulation(z, idx, idx, sink.astype(np.float32))
    with pytest.raises(ValueError):
        H.plot_flow_indicator(z, max_pool_kernel=2.0)
    for fn in fns:                                           # valid arguments, no CUDA device
        with pytest.raises(L.TdxError):
            fn(z)
    with pytest.raises(L.TdxError):
        H.plot_flow_indicator(z, max_pool_kernel=100)        # larger than the image: an empty result, not an error


def test_bench_hydrology_help_runs():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_hydrology.py"), "--help"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--iters" in out.stdout and "--sizes" in out.stdout and "--serpentine" in out.stdout
