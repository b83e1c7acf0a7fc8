"""Depression fill and river-bed smoothing on the GPU (csrc/tdx_depress.cu through
terrain_diffusion_b200.inference.hydrology): every golden of the reference's own fill_depressions_priority_flood /
smooth_river_bumps (tests/golden/depressions_golden.npz), the oracle at 1024^2, routing a filled window, the
adversarial serpentine flat, input kinds, in-place writes, determinism, streams and devices.

Tolerances: the fill is bit-identical (the relaxation's fixed point does not depend on the thread schedule); the
counts of a filled window are bit-identical and its indicator within 1 ulp (numpy's fp32 log1p); the smoothing is
bit-identical to the oracle and within the CPU test's stated bound of the reference goldens."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import depressions as O
from terrain_diffusion_b200.inference import (d8_flow, fill_depressions_priority_flood, flow_accumulation,
                                              plot_flow_indicator, smooth_river_bumps)
from terrain_diffusion_b200.inference import hydrology as H
from tests._depression_inputs import (FILL_CASES, SMOOTH_CASES, composition_case, fill_case, fill_serpentine,
                                      smooth_case)
from tests._hydrology_inputs import smooth_field
from tests.test_depressions_cpu import same_bits, smooth_within_bound
from tests.test_hydrology_cpu import ulps

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "depressions_golden.npz")


def bits(x):
    x = x.cpu().numpy() if isinstance(x, torch.Tensor) else x
    return x.view(np.uint8).tobytes() + str((x.dtype, x.shape)).encode()


def same_bits_nan_by_position(a, b) -> bool:
    """Bit-identical except that NaN is compared by position: a NaN made by arithmetic (an +inf pixel's Laplacian)
    has the device's canonical bits on the GPU and the x86 default NaN on the host."""
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and same_bits(np.where(nan, 0, a).astype(np.float32),
                                                                               np.where(nan, 0, b).astype(np.float32))


@pytest.mark.parametrize("name", list(FILL_CASES))
def test_fill_matches_reference_golden(name):
    z, kw = fill_case(name)
    got = fill_depressions_priority_flood(z, **kw)
    assert same_bits(got, G[f"fill.{name}"])


@pytest.mark.parametrize("n,connectivity", [(1024, 8), (333, 4), (333, 8)])
def test_fill_matches_oracle(n, connectivity):
    z = smooth_field(n, seed=21, ocean_fraction=0.05)
    z[z > np.nanquantile(z, 0.9)] = np.inf                   # +inf land among the peaks
    ref, oracle_passes = O.fill(z, connectivity=connectivity)
    zd = torch.from_numpy(z).cuda()
    out, passes = H._fill(zd, float(np.float32(1e-3)), connectivity, float("nan"))
    assert same_bits(out.cpu().numpy(), ref) and (ref > z).sum() > 100
    assert 1 <= passes <= oracle_passes                      # tiles converge locally: never more passes than Jacobi


def test_fill_then_route_matches_reference_golden():
    z = composition_case()
    filled = fill_depressions_priority_flood(z)
    assert same_bits(filled, G["compose.filled"])
    rr, cc, is_sink, _ = d8_flow(filled)
    assert same_bits(flow_accumulation(filled, rr, cc, is_sink), G["compose.A"])
    ind = plot_flow_indicator(fill_depressions_priority_flood(torch.from_numpy(z).cuda())).cpu().numpy()
    assert ind.shape == G["compose.ind1"].shape and ulps(ind, G["compose.ind1"]) <= 1


def test_serpentine_flat_single_long_chain():
    n = 512
    z, chain = fill_serpentine(n)
    assert chain > n * n // 2 - 2 * n
    ref = O.fill_ordered(z)
    zd = torch.from_numpy(z).cuda()
    out, passes = H._fill(zd, float(np.float32(1e-3)), 8, float("nan"))
    got = out.cpu().numpy()
    assert same_bits(got, ref)
    assert float(got[z == 100.0].max()) > 100.0 + 0.9e-3 * chain * 0.9   # every chain cell raised past the last
    assert passes > n                                          # the chain crosses a tile boundary on every row


@pytest.mark.parametrize("name", list(SMOOTH_CASES))
def test_smooth_matches_oracle_and_reference_golden(name):
    z, kw = smooth_case(name)
    got = smooth_river_bumps(z, **kw)
    assert same_bits(got, O.smooth(z, **kw))
    assert smooth_within_bound(got, G[f"smooth.{name}"], z)


def test_smooth_large_window_matches_oracle():
    z = smooth_field(1024, seed=23)
    z[7, 3] = np.inf                                          # spreads NaN through the Laplacian
    for kw in ({}, {"slope_thresh": 20, "smooth_strength": 0.1, "iterations": 4}):
        got, ref = smooth_river_bumps(torch.from_numpy(z).cuda(), **kw).cpu().numpy(), O.smooth(z, **kw)
        assert np.isnan(ref).sum() > np.isnan(z).sum() and same_bits_nan_by_position(got, ref)


def test_input_kinds_in_place_and_repeats_give_identical_bits():
    z = smooth_field(300, seed=24)
    zd = torch.from_numpy(z).cuda()
    ref = fill_depressions_priority_flood(z)
    runs = [fill_depressions_priority_flood(x) for x in (torch.from_numpy(z), zd, zd, z.astype(np.float64))]
    assert runs[1].is_cuda and runs[1].dtype == torch.float32 and isinstance(runs[0], np.ndarray)
    assert all(bits(r) == bits(ref) for r in runs)
    assert np.array_equal(zd.cpu().numpy(), z, equal_nan=True)          # the input is not touched
    # in_place: a float32 array or tensor receives the result and is returned; other dtypes are left alone
    a = z.copy()
    assert fill_depressions_priority_flood(a, in_place=True) is a and bits(a) == bits(ref)
    t = zd.clone()
    assert fill_depressions_priority_flood(t, in_place=True) is t and bits(t) == bits(ref)
    tc = torch.from_numpy(z.copy())
    back = fill_depressions_priority_flood(tc, in_place=True)
    assert isinstance(back, np.ndarray) and bits(tc) == bits(ref) and bits(back) == bits(ref)
    big = torch.full((300, 600), 7.0, device="cuda")
    view = big[:, ::2]                                                  # non-contiguous
    view.copy_(zd)
    fill_depressions_priority_flood(view, in_place=True)
    assert bits(view.contiguous()) == bits(ref) and bool((big[:, 1::2] == 7.0).all())
    a64 = z.astype(np.float64)
    out64 = fill_depressions_priority_flood(a64, in_place=True)
    assert out64 is not a64 and np.array_equal(a64, z.astype(np.float64), equal_nan=True) and bits(out64) == bits(ref)
    sref = smooth_river_bumps(z)
    for x in (torch.from_numpy(z), zd, zd, z.astype(np.float64)):
        assert bits(smooth_river_bumps(x)) == bits(sref)


def test_side_stream_and_second_device():
    z = smooth_field(512, seed=25)
    ref, sref = fill_depressions_priority_flood(z), smooth_river_bumps(z)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        zd = torch.from_numpy(z).cuda(non_blocking=False)
        out = fill_depressions_priority_flood(zd)
        sm = smooth_river_bumps(zd)
    s.synchronize()
    assert bits(out) == bits(ref) and bits(sm) == bits(sref)
    if torch.cuda.device_count() < 2:
        pytest.skip("second device: only one CUDA device visible")
    z1 = torch.from_numpy(z).to("cuda:1")
    out1, sm1 = fill_depressions_priority_flood(z1), smooth_river_bumps(z1)
    assert out1.device == z1.device and sm1.device == z1.device
    assert bits(out1) == bits(ref) and bits(sm1) == bits(sref)
