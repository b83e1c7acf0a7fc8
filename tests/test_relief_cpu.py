"""Shaded relief map, CPU side: the oracle restatement (oracle/relief.py) against the golden vectors recorded from the
reference's own get_relief_map (tests/golden/make_golden_relief.py), the host pieces of
terrain_diffusion_b200.inference.relief (filter taps, NaN-median fill, argument checks) and the pipeline wiring."""
import subprocess
import sys
import warnings
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import relief as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import relief as R
from tests._relief_inputs import CASES, golden_stride, relief_case

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "relief_golden.npz")


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(name):
    elev, kw = relief_case(name)
    with np.errstate(invalid="ignore"):
        full = O.relief_map(elev, **kw)
    assert full.shape == elev.shape + (3,) and full.dtype == np.float32
    s = golden_stride(name)
    got, g = full[::s, ::s], G[name]
    assert got.shape == g.shape
    assert np.array_equal(np.isnan(got), np.isnan(g))
    fin = ~np.isnan(g)
    assert float(np.abs(got[fin] - g[fin]).max()) <= 1e-6


def test_golden_cases_cover_the_branches():
    # nan: NaN pixels filled with a negative median come out ocean-coloured (the reference's quirk), none stay NaN
    elev, _ = relief_case("nan")
    n = int(np.isnan(elev).sum())
    assert n % 2 == 0 and (elev.size - n) % 2 == 0 and np.nanmedian(elev) < 0
    assert not np.isnan(G["nan"]).any()
    # vrange: land below vmin gives norm < 0, norm ** 0.7 = NaN and the colormap's bad colour, i.e. black
    elev, kw = relief_case("vrange")
    s = golden_stride("vrange")
    below = (elev > 0) & (elev < kw["vmin"])
    assert below[::s, ::s].any() and np.all(G["vrange"][below[::s, ::s]] == 0)
    assert np.all(relief_case("ocean")[0] < 0) and np.all(relief_case("land")[0] > 0)


def test_terrain_lut_endpoints_and_stops():
    lut = R.terrain_lut()
    assert lut.shape == (256, 3) and lut.dtype == np.float64
    assert np.array_equal(lut[0], [0.2, 0.2, 0.6]) and np.array_equal(lut[255], [1.0, 1.0, 1.0])
    assert np.all(np.diff(lut[64:128, 0]) > 0)           # 0.25 .. 0.5: green (0, 0.8, 0.4) towards (1, 1, 0.6)
    rgba = O.terrain_cmap(np.array([0.0, 1.0, -0.1, 1.5, np.nan, 0.5], np.float32))
    assert np.array_equal(rgba[:, :3], np.stack([lut[0], lut[255], lut[0], lut[255], np.zeros(3), lut[128]]))


@pytest.mark.parametrize("sigma", [6.0, 1.2, 0.8, 3.0, 0.3])
def test_gaussian_taps_are_scipys(sigma):
    from scipy.ndimage import gaussian_filter1d
    taps = R.gaussian_taps(sigma)
    r = len(taps) // 2
    assert r == int(4 * sigma + 0.5) and np.array_equal(taps, taps[::-1])
    delta = np.zeros(2 * r + 1 + 2 * r)
    delta[2 * r] = 1.0                                      # the impulse response of scipy's filter is its taps, exactly
    assert np.array_equal(gaussian_filter1d(delta, sigma)[r:3 * r + 1], taps)


def test_nanmedian_fill_is_numpys():
    rng = np.random.RandomState(0)
    for n, n_nan in ((10, 3), (11, 4), (3072, 150), (7, 0), (5, 5), (1, 0), (2, 1)):
        x = (rng.randn(n) * 300 - 100).astype(np.float32)
        x[rng.choice(n, n_nan, replace=False)] = np.nan
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)      # all-NaN slice
            m = np.nanmedian(x)
        ref = float(m) if np.isfinite(m) else 0.0
        assert R.nanmedian_fill(torch.from_numpy(x)) == ref, (n, n_nan)
    assert R.nanmedian_fill(torch.tensor([1.0, np.inf, np.inf, np.nan])) == 0.0


def test_argument_errors_come_before_any_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(R, "_relief", no_device)
    monkeypatch.setattr(L, "lib", no_device)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    e = np.zeros((8, 8), np.float32)
    with pytest.raises(NotImplementedError):
        R.get_relief_map(e, None, e, None)
    with pytest.raises(NotImplementedError):
        R.get_relief_map(e, None, None, e)
    with pytest.raises(NotImplementedError):
        R.get_relief_map(e, None, None, None, rgb=np.zeros((8, 8, 3)))
    for shape in ((8,), (1, 8), (8, 1), (2, 3, 4), (0, 5)):
        with pytest.raises(ValueError):
            R.get_relief_map(np.zeros(shape, np.float32), None, None, None)
    with pytest.raises(ValueError):
        R.get_relief_map(torch.zeros(1, 16), None, None, None)
    with pytest.raises(ValueError):
        R.get_relief_map(e, None, None, None, sigma_large=30.0)
    with pytest.raises(L.TdxError):                          # valid arguments, no CUDA device
        R.get_relief_map(e, np.zeros((3, 8, 8)), None, None)


def test_world_pipeline_get_relief_wiring(monkeypatch):
    from terrain_diffusion_b200.inference.pipeline import WorldPipeline
    calls = {}

    def fake_relief(elev, climate, biome, flow, **kw):
        calls["args"] = (elev, climate, biome, flow, kw)
        return torch.ones(2, 3, 3)

    monkeypatch.setattr(R, "get_relief_map", fake_relief)
    p = WorldPipeline(native_resolution=30.0)
    p.get_elev = lambda i1, j1, i2, j2: ("ELEV", i1, j1, i2, j2)
    out = p.get_relief(1, 2, 3, 5, relief=0.7)
    assert isinstance(out, np.ndarray) and out.shape == (2, 3, 3)
    assert calls["args"] == (("ELEV", 1, 2, 3, 5), None, None, None, {"relief": 0.7, "resolution": 30.0})
    p._host_views = False                                     # TerrainPipeline: the device tensor itself
    assert torch.is_tensor(p.get_relief(0, 0, 2, 3, resolution=90))
    assert calls["args"][4] == {"resolution": 90}


def test_bench_relief_help_runs():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_relief.py"), "--help"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--iters" in out.stdout and "--sizes" in out.stdout
