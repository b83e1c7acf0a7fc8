"""River routing on the GPU (csrc/tdx_hydro.cu through terrain_diffusion_b200.inference.hydrology): every golden of the
reference's own d8_flow / flow_accumulation / plot_flow_indicator (tests/golden/hydrology_golden.npz) and the oracle at
1024^2, the adversarial serpentine path, a full check of a 4096^2 (2^24 px) accumulation, input kinds, determinism,
streams and devices, and the receiver checks of flow_accumulation.

Tolerance: kmax, rr, cc, is_sink and A are bit-identical (the counts are exact integers under any thread schedule);
the indicator is within 1 ulp, because numpy's fp32 log1p depends on the host's SIMD path."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import hydrology as O
from terrain_diffusion_b200.inference import d8_flow, flow_accumulation, plot_flow_indicator
from tests._hydrology_inputs import CASES, hydrology_case, serpentine, smooth_field
from tests.test_hydrology_cpu import ulps

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "hydrology_golden.npz")


def bits(x):
    x = x.cpu().numpy() if isinstance(x, torch.Tensor) else x
    return x.view(np.uint8).tobytes() + str((x.dtype, x.shape)).encode()


def check_against_oracle(z, tol=1e-3, pools=(1,)):
    rr, cc, is_sink, kmax = d8_flow(z, tol=tol)
    orr, occ, osink, okmax = O.d8(z, tol)
    assert rr.dtype == cc.dtype == kmax.dtype == np.int64 and is_sink.dtype == bool
    assert np.array_equal(kmax, okmax) and np.array_equal(rr, orr) and np.array_equal(cc, occ)
    assert np.array_equal(is_sink, osink)
    a = flow_accumulation(z, rr, cc, is_sink)
    oa = O.accumulate(z, orr, occ, osink)
    assert a.dtype == np.float32 and np.array_equal(a.view(np.uint32), oa.view(np.uint32))
    for k in pools:
        ind = plot_flow_indicator(z, max_pool_kernel=k)
        ref = O.flow_indicator(z, k)                            # the indicator routes with the default tol
        assert ind.dtype == np.float32 and ind.shape == ref.shape and ulps(ind, ref) <= 1
    return kmax, is_sink, a


@pytest.mark.parametrize("name", list(CASES))
def test_matches_reference_golden(name):
    z, tol, pools = hydrology_case(name)
    kmax, is_sink, a = check_against_oracle(z, tol, pools)
    assert np.array_equal(kmax, G[f"{name}.kmax"]) and np.array_equal(is_sink, G[f"{name}.is_sink"])
    assert np.array_equal(a.view(np.uint32), G[f"{name}.A"].view(np.uint32))
    for k in pools:
        ind, g = plot_flow_indicator(z, max_pool_kernel=k), G[f"{name}.ind{k}"]
        assert ind.shape == g.shape and ulps(ind, g) <= 1


@pytest.mark.parametrize("n", [1024, 333])
def test_smooth_terrain_matches_oracle(n):
    z = smooth_field(n, seed=7)
    _, _, a = check_against_oracle(z, pools=(1, 2, 8))
    assert a.max() > 1000


def test_serpentine_single_long_path():
    n = 256
    z, path = serpentine(n)
    rr, cc, is_sink, kmax = d8_flow(z)
    a = flow_accumulation(z, rr, cc, is_sink)
    oa = O.accumulate(z, rr, cc, is_sink)
    assert len(path) == 32895 and a.ravel()[path[-1]] == n * n
    assert np.array_equal(a.view(np.uint32), oa.view(np.uint32))
    assert ulps(plot_flow_indicator(z), np.log1p(oa)) <= 1


def test_full_2_24_pixel_accumulation_satisfies_the_tree_sum():
    """At 4096^2 the accumulation is checked through its defining identity, which has one solution on a forest:
    A[v] == 1 + sum of A over the pixels draining into v for valid v, A == 0 elsewhere."""
    z = smooth_field(4096, seed=11)
    zd = torch.from_numpy(z).cuda()
    rr, cc, is_sink, kmax = d8_flow(zd)
    a = flow_accumulation(zd, rr, cc, is_sink).cpu().numpy().ravel()
    rr, cc, is_sink = rr.cpu().numpy(), cc.cpu().numpy(), is_sink.cpu().numpy()
    orr, occ, osink, okmax = O.d8(z)
    assert np.array_equal(kmax.cpu().numpy(), okmax) and np.array_equal(rr, orr) and np.array_equal(cc, occ)
    assert np.array_equal(is_sink, osink)
    recv = O.receivers(z, rr, cc, is_sink)
    src = np.flatnonzero(recv >= 0)
    valid = ~O.ocean(z).ravel()
    inflow = np.bincount(recv[src], weights=a[src].astype(np.float64), minlength=a.size)
    assert np.all(a[~valid] == 0)
    assert np.array_equal(a[valid].astype(np.float64), 1.0 + inflow[valid])
    assert a.max() > 1000 and a.sum() > valid.sum()
    ind = plot_flow_indicator(zd, max_pool_kernel=8).cpu().numpy()
    ref = O.indicator(a.reshape(z.shape), z, 8)
    assert ulps(ind, ref) <= 1


def test_input_kinds_and_repeats_give_identical_bits():
    z = smooth_field(512, seed=3)
    zd = torch.from_numpy(z).cuda()
    host = d8_flow(z)
    for other in (d8_flow(torch.from_numpy(z)), d8_flow(zd), d8_flow(zd)):
        assert all(bits(x) == bits(y) for x, y in zip(other, host))
    dev = d8_flow(zd)
    assert dev[0].is_cuda and dev[2].dtype == torch.bool and dev[3].dtype == torch.int64
    a = flow_accumulation(z, *host[:3])
    runs = [flow_accumulation(zd, *dev[:3]) for _ in range(3)] + [flow_accumulation(torch.from_numpy(z), *host[:3])]
    runs.append(flow_accumulation(zd, *host[:3]))               # host receivers, device elevation
    assert runs[0].is_cuda and all(bits(r) == bits(a) for r in runs)
    ind = plot_flow_indicator(z, 3)
    assert all(bits(plot_flow_indicator(x, 3)) == bits(ind) for x in (zd, zd, torch.from_numpy(z)))
    # a float64 z is computed in fp32
    assert bits(plot_flow_indicator(z.astype(np.float64), 3)) == bits(ind)


def test_side_stream_and_second_device():
    z = smooth_field(512, seed=5)
    ref = plot_flow_indicator(z)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        zd = torch.from_numpy(z).cuda(non_blocking=False)
        out = plot_flow_indicator(zd)
        rr, cc, sink, _ = d8_flow(zd)
        a = flow_accumulation(zd, rr, cc, sink)
    s.synchronize()
    assert bits(out) == bits(ref) and bits(a) == bits(flow_accumulation(z, *d8_flow(z)[:3]))
    if torch.cuda.device_count() < 2:
        pytest.skip("second device: only one CUDA device visible")
    z1 = torch.from_numpy(z).to("cuda:1")
    out1 = plot_flow_indicator(z1)
    assert out1.device == z1.device and bits(out1) == bits(ref)
    rr1, cc1, sink1, _ = d8_flow(z1)
    assert rr1.device == z1.device and bits(flow_accumulation(z1, rr1, cc1, sink1)) == bits(a)


def test_flow_accumulation_rejects_receivers_the_reference_would_order_arbitrarily():
    z = np.array([[5.0, 5.0, 4.0], [6.0, 3.0, -1.0]], np.float32)
    rr, cc = np.indices(z.shape)                                # every pixel its own receiver, all sinks but (0, 0)
    sink = np.ones(z.shape, bool)
    sink[0, 0] = False

    def route(target, zz=z):
        r, c = rr.copy(), cc.copy()
        r[0, 0], c[0, 0] = target
        return flow_accumulation(zz, r, c, sink)

    for target in ((0, 0), (0, 1), (1, 0)):                     # itself, level, uphill
        with pytest.raises(ValueError, match="strictly"):
            route(target)
    with pytest.raises(ValueError, match="strictly"):          # the same on the device, receivers from the host
        flow_accumulation(torch.from_numpy(z).cuda(), torch.tensor([[0, 0, 0], [1, 1, 1]]).cuda(), cc, sink)
    for target in ((2, 0), (0, 3), (-1, 0)):
        with pytest.raises(ValueError, match="outside"):
            route(target)
    assert np.array_equal(route((1, 1)), [[1, 1, 1], [1, 2, 0]])   # downhill: followed
    assert np.array_equal(route((1, 2)), [[1, 1, 1], [1, 1, 0]])   # into the ocean: not followed, no check
    level = z.copy()
    level[0, 1] = np.nan                                            # an invalid target is not followed either
    assert np.array_equal(route((0, 1), level), [[1, 0, 1], [1, 1, 0]])


def test_infinite_elevation_on_the_device_is_an_error():
    z = smooth_field(64, seed=2)
    z[10, 10] = np.inf
    zd = torch.from_numpy(z).cuda()
    for fn in (d8_flow, plot_flow_indicator):
        with pytest.raises(ValueError, match="inf"):
            fn(zd)
    with pytest.raises(ValueError, match="inf"):
        flow_accumulation(zd, *[torch.zeros(64, 64, dtype=torch.int64, device="cuda")] * 2,
                          torch.ones(64, 64, dtype=torch.bool, device="cuda"))


def test_neg_inf_ocean_routes_after_the_fill():
    from terrain_diffusion_b200.inference import fill_depressions_priority_flood
    from tests._hydrology_inputs import FILLED_CASES
    for name, (build, pools) in FILLED_CASES.items():
        z = build()
        filled = fill_depressions_priority_flood(z)
        assert np.isneginf(filled).any()
        assert np.array_equal(filled.view(np.uint32), G[f"{name}.filled"].view(np.uint32))
        rr, cc, is_sink, kmax = d8_flow(filled)
        assert np.array_equal(kmax, G[f"{name}.kmax"]) and np.array_equal(is_sink, G[f"{name}.is_sink"])
        a = flow_accumulation(filled, rr, cc, is_sink)
        assert np.array_equal(a.view(np.uint32), G[f"{name}.A"].view(np.uint32))
        for k in pools:
            ind = plot_flow_indicator(fill_depressions_priority_flood(torch.from_numpy(z).cuda()), max_pool_kernel=k)
            assert ulps(ind.cpu().numpy(), G[f"{name}.ind{k}"]) <= 1
