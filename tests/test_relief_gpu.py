"""Shaded relief map on the GPU (csrc/tdx_relief.cu through terrain_diffusion_b200.inference.get_relief_map): the
filter against scipy bit for bit, every golden of the reference's own get_relief_map (tests/golden/relief_golden.npz),
the CUDA-tensor path against the numpy path, and WorldPipeline.get_relief.

Tolerance: the NaN pattern is identical; every other value is within 2e-5 of the golden, except that a land pixel may
take the adjacent colormap entry where the oracle's fp32 colormap argument x 256 lies within 1e-4 of an integer (the
device's fp32 power may round the other way there).  The goldens of the larger cases hold every other row and column,
so the full image is also held to the same rule against the oracle, which is pinned to the golden pixels.  Each case
prints its count of such pixels and its worst share of the 2e-5 bound.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter as scipy_gaussian_filter

from oracle import relief as O
from oracle import unet as ounet
from terrain_diffusion_b200.inference import TerrainPipeline, get_relief_map
from terrain_diffusion_b200.inference import relief as R
from terrain_diffusion_b200.models import EDMUnet2D
from tests._post_inputs import field
from tests._relief_contract import TOL, compare
from tests._relief_inputs import CASES, golden_stride, relief_case
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu
G = np.load(Path(__file__).resolve().parent / "golden" / "relief_golden.npz")


@pytest.mark.parametrize("shape", [(2, 2), (5, 7), (33, 17), (129, 65), (1024, 1024)])
def test_gaussian_filter_is_scipy_bit_for_bit(shape):
    x = field(shape[0] * 31 + shape[1], *shape, 100.0, 500.0)
    xd = torch.from_numpy(x).cuda()
    for s in (6.0, 1.2, 0.8, 3.0):
        got = R.gaussian_filter(xd, [s])[0].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), scipy_gaussian_filter(x, s).view(np.uint32)), (shape, s)
    both = R.gaussian_filter(xd, [6.0, 1.2]).cpu().numpy()
    assert np.array_equal(both[0], scipy_gaussian_filter(x, 6.0)) and np.array_equal(both[1], scipy_gaussian_filter(x, 1.2))


@pytest.mark.parametrize("name", list(CASES))
def test_public_function_matches_reference_golden(name):
    elev, kw = relief_case(name)
    got = get_relief_map(elev, None, None, None, **kw)
    assert isinstance(got, np.ndarray) and got.shape == elev.shape + (3,)
    with np.errstate(invalid="ignore"):
        parts = O.relief_parts(elev, **kw)
    s = golden_stride(name)
    n_boundary, share = compare(got[::s, ::s], G[name], {k: v[::s, ::s] for k, v in parts.items()})
    n_full, share_full = compare(got, parts["rgb"], parts)
    print(f"\nrelief {name}: vs golden (every {s}. pixel) {n_boundary} LUT-boundary pixels, worst share of the "
          f"{TOL:g} bound {share:.3f}; vs oracle (all pixels) {n_full}, {share_full:.3f}")


def test_cuda_path_is_the_numpy_path_and_repeatable():
    for name in ("mixed", "nan", "vrange"):
        elev, kw = relief_case(name)
        host = get_relief_map(elev, None, None, None, **kw)
        d = torch.from_numpy(elev).cuda()
        a = get_relief_map(d, None, None, None, **kw)
        b = get_relief_map(d, None, None, None, **kw)
        assert a.is_cuda and a.dtype == torch.float32 and tuple(a.shape) == elev.shape + (3,)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        assert np.array_equal(a.cpu().numpy().view(np.uint32), host.view(np.uint32))
        assert np.array_equal(get_relief_map(torch.from_numpy(elev), None, None, None, **kw).view(np.uint32),
                              host.view(np.uint32))                            # CPU tensor in, numpy out


def test_nan_on_land_stays_nan_and_matches_oracle():
    """NaN pixels whose fill (the NaN-median) is above sea level stay NaN; an all-NaN window fills with 0."""
    elev = field(50, 48, 40, 600.0, 200.0)
    elev[5:9, 3:30] = np.nan
    elev[20, 20] = np.nan                                     # odd NaN count: the median is one value
    got = get_relief_map(elev, None, None, None)
    ref = O.relief_map(elev)
    assert np.isnan(got[5:9, 3:30]).all() and np.array_equal(np.isnan(got), np.isnan(ref))
    fin = ~np.isnan(ref)
    assert float(np.abs(got[fin] - ref[fin]).max()) <= TOL
    allnan = np.full((6, 9), np.nan, np.float32)
    assert np.isnan(get_relief_map(allnan, None, None, None)).all()


def test_terrain_pipeline_get_relief_is_get_elev_then_relief():
    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.cuda()

    def cond_fn(i1, i2, j1, j2):
        gg = torch.Generator().manual_seed(i1 * 7919 + j1 + 12345)
        return torch.randn(5, i2 - i1, j2 - j1, generator=gg)

    g = torch.Generator().manual_seed(3)
    pipe = TerrainPipeline(build(COARSE_CFG), build(BASE_CFG), build(ounet.DECODER_CFG), seed=7, conditioning_fn=cond_fn,
                           coarse_means=(torch.randn(6, generator=g) * 0.1).tolist(),
                           coarse_stds=(torch.rand(6, generator=g) + 0.5).tolist(), cond_snr=[0.3, 0.5, 1.0, 2.0, 4.0],
                           histogram_raw=torch.randn(5, generator=g), latents_means=torch.zeros(7),
                           latents_stds=torch.ones(7), decoder_tile_size=128, decoder_tile_stride=96,
                           residual_mean=0.1, residual_std=1.2, native_resolution=30.0)
    window = (-20, 10, 44, 90)
    got = pipe.get_relief(*window)
    ref = get_relief_map(pipe.get_elev(*window), None, None, None, resolution=pipe.native_resolution)
    assert got.is_cuda and tuple(got.shape) == (64, 80, 3)
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))
    assert torch.isfinite(got).all() and float(got.min()) >= 0 and float(got.max()) <= 1
