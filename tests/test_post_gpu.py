"""Post step (elevation read-out) on the GPU: every tdx_post_* / tdx_resize_aa_axis / tdx_gaussian_blur primitive and
their composition (terrain_diffusion_b200/inference/postproc.py) against the CPU oracle and against the golden vectors
recorded from the reference (tests/golden/post_golden.npz, post_coastal_golden.npz).

Tolerance: the kernels use the oracle's operation order with explicitly rounded fp32 operations, so primitives agree to
a few ulp (rtol 2e-6 of the tensor's max); against the reference goldens 1e-5 (torch's conv sums in another order)."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import postproc as P
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import postproc as H
from tests._post_inputs import (COASTAL_SCALE, COASTAL_WINDOW, ELEV_WINDOWS, RESIDUAL_MEAN, RESIDUAL_STD,
                                coarse_canvas, coastal_canvas, coastal_elev, elev_canvases, field, laplacian_case)

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "post_golden.npz")
GC = np.load(Path(__file__).resolve().parent / "golden" / "post_coastal_golden.npz")


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("shape,size", [((12, 10), (96, 80)), ((96, 80), (12, 10)), ((14, 12), (112, 96)), ((37, 53), (9, 11)),
                                        ((64, 136), 17), ((96, 80), 10), ((20, 20), (20, 45)), ((31, 17), (64, 17))])
def test_resize_matches_oracle(shape, size):
    x = field(7, *shape, 0.0, 2.0)
    got = H.resize_bilinear(dev(x), size).cpu().numpy()
    ref = P.resize_bilinear(x, size)
    assert got.shape == ref.shape
    assert rel(got, ref) < 2e-6


def test_pad_blur_and_extrapolated_resize_match_oracle():
    x = field(3, 13, 9, 1.0, 2.0)
    assert np.array_equal(H.pad_linear_extrapolation(dev(x)).cpu().numpy(), P.pad_linear_extrapolation(x))
    one = field(4, 1, 7)
    assert np.array_equal(H.pad_linear_extrapolation(dev(one)).cpu().numpy(), P.pad_linear_extrapolation(one))
    assert rel(H.resize_extrapolated(dev(x), (104, 72)).cpu().numpy(), P.resize_extrapolated(x, (104, 72))) < 2e-6
    y = field(5, 17, 36, -30.0, 40.0)
    assert rel(H.gaussian_blur(dev(y), 11, 5.0).cpu().numpy(), P.gaussian_blur(y, 11, 5.0)) < 2e-6
    assert rel(H.gaussian_blur(dev(y), 3, 0.8).cpu().numpy(), P.gaussian_blur(y, 3, 0.8)) < 2e-6
    with pytest.raises(L.TdxError):
        H.gaussian_blur(dev(field(6, 5, 20)), 11, 5.0)          # reflect padding 5 needs more than 5 rows


@pytest.mark.parametrize("name", ["rect", "square", "wide"])
def test_laplacian_functions_match_reference_golden(name):
    r, l = laplacian_case(name)
    rd, ld = dev(r), dev(l)
    assert rel(H.laplacian_decode(rd, ld, extrapolate=True).cpu().numpy(), G[f"lap_{name}_decode_extrap"]) < 1e-5
    _, l2 = H.laplacian_denoise(rd, ld, 5)
    assert tuple(l2.shape) == G[f"lap_{name}_lowres"].shape
    assert rel(l2.cpu().numpy(), G[f"lap_{name}_lowres"]) < 1e-5
    assert rel(H.laplacian_decode(rd, l2).cpu().numpy(), G[f"lap_{name}_elev"]) < 1e-5
    assert rel(l2.cpu().numpy(), P.laplacian_denoise(r, l, 5)[1]) < 2e-6


class CudaCanvas:
    def __init__(self, fake):
        self.fake = fake

    def __getitem__(self, key):
        _, ys, xs = key
        return dev(self.fake.planes(ys.start, ys.stop, xs.start, xs.stop))


@pytest.mark.parametrize("name", list(ELEV_WINDOWS))
def test_compute_elev_matches_reference_golden_and_packs_int16(name):
    resid, lat = elev_canvases()
    i1, j1, i2, j2 = ELEV_WINDOWS[name]
    elev, i16 = H.compute_elev(CudaCanvas(resid), CudaCanvas(lat), i1, j1, i2, j2, 8, RESIDUAL_MEAN, RESIDUAL_STD,
                               as_int16=True)
    e = elev.cpu().numpy()
    g = G[f"elev_{name}"]
    assert e.shape == g.shape
    assert rel(e, g) < 1e-5
    ref = P.compute_elev(i1, j1, i2, j2, resid.planes, lat.planes, 8, RESIDUAL_MEAN, RESIDUAL_STD)
    assert rel(e, ref) < 2e-6
    assert i16.dtype == torch.int16 and np.array_equal(i16.cpu().numpy(), P.elev_to_int16(e))
    only = H.compute_elev(CudaCanvas(resid), CudaCanvas(lat), i1, j1, i2, j2, 8, RESIDUAL_MEAN, RESIDUAL_STD)
    assert torch.equal(only, elev)
    with pytest.raises(ValueError):
        H.compute_elev(CudaCanvas(resid), CudaCanvas(lat), i2, j1, i1, j2, 8, RESIDUAL_MEAN, RESIDUAL_STD)


@pytest.mark.parametrize("name", list(ELEV_WINDOWS))
def test_compute_climate_matches_reference_golden(name):
    """tdx_lapse_rate + tdx_climate_sample = WorldPipeline._compute_climate (world_pipeline.py:1314-1365)."""
    i1, j1, i2, j2 = ELEV_WINDOWS[name]
    cc = coarse_canvas()
    elev = G[f"elev_{name}"]
    got = H.compute_climate(CudaCanvas(cc), i1, j1, i2, j2, dev(elev), 8).cpu().numpy()
    ref = P.compute_climate(i1, j1, i2, j2, elev, cc.planes, 8)
    g = G[f"climate_{name}"]                               # reference, stored at every other pixel
    assert got.shape == ref.shape == (5, i2 - i1, j2 - j1)
    for k in range(5):
        assert rel(got[k], ref[k]) < 2e-6, k
        assert rel(got[k, ::2, ::2], g[k]) < 1e-5, k
    with pytest.raises(ValueError):
        H.compute_climate(CudaCanvas(cc), i1, j1, i2 + 1, j2, dev(elev), 8)


def test_compute_climate_coastal_matches_reference_golden():
    """A coastal window at scale 2 whose lapse-rate regressions take every branch (all-ocean and sparse-land fallbacks,
    flat land, both clip bounds): bit for bit against the oracle, and against the reference's own result."""
    i1, j1, i2, j2 = COASTAL_WINDOW
    cc, elev = coastal_canvas(), coastal_elev()
    got = H.compute_climate(CudaCanvas(cc), i1, j1, i2, j2, dev(elev), COASTAL_SCALE).cpu().numpy()
    ref = P.compute_climate(i1, j1, i2, j2, elev, cc.planes, COASTAL_SCALE)
    assert got.shape == ref.shape == (5, i2 - i1, j2 - j1)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    g = GC["climate"]                                      # reference, stored at every fourth pixel
    for k in range(5):
        assert rel(got[k, ::4, ::4], g[k]) < 1e-5, k
