"""Post step (elevation read-out), CPU side: the oracle restatement against the golden vectors recorded from the
reference's own laplacian_encoder.py / WorldPipeline._compute_elev (tests/golden/make_golden_post.py), and the integer
window geometry of the product host code against the oracle."""
from pathlib import Path

import numpy as np
import pytest

from oracle import postproc as P
from tests._post_inputs import (COASTAL_SCALE, COASTAL_WINDOW, ELEV_WINDOWS, RESIDUAL_MEAN, RESIDUAL_STD, coarse_canvas,
                                coastal_canvas, coastal_coarse_map, coastal_elev, elev_canvases, laplacian_case)

G = np.load(Path(__file__).resolve().parent / "golden" / "post_golden.npz")
GC = np.load(Path(__file__).resolve().parent / "golden" / "post_coastal_golden.npz")


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


@pytest.mark.parametrize("name", ["rect", "square", "wide"])
def test_oracle_laplacian_functions_match_reference_golden(name):
    r, l = laplacian_case(name)
    assert rel(P.laplacian_decode(r, l, extrapolate=True), G[f"lap_{name}_decode_extrap"]) < 2e-6
    _, l2 = P.laplacian_denoise(r, l, 5)
    # an int size means "shorter edge": the non-square cases come out with the reference's (distorted) low-res shape
    assert l2.shape == G[f"lap_{name}_lowres"].shape
    assert rel(l2, G[f"lap_{name}_lowres"]) < 2e-6
    assert rel(P.laplacian_decode(r, l2), G[f"lap_{name}_elev"]) < 2e-6


@pytest.mark.parametrize("name", list(ELEV_WINDOWS))
def test_oracle_compute_elev_matches_reference_golden(name):
    resid, lat = elev_canvases()
    i1, j1, i2, j2 = ELEV_WINDOWS[name]
    e = P.compute_elev(i1, j1, i2, j2, resid.planes, lat.planes, 8, RESIDUAL_MEAN, RESIDUAL_STD)
    g = G[f"elev_{name}"]
    assert e.shape == g.shape == (i2 - i1, j2 - j1)
    assert rel(e, g) < 2e-6
    i16 = P.elev_to_int16(g)
    assert i16.dtype == np.dtype("<i2") and int(i16.max()) <= 32767 and np.array_equal(i16, np.floor(g).astype(np.int16))


def test_padded_window_integer_geometry_is_identical_in_product_and_oracle():
    from terrain_diffusion_b200.inference import postproc as H
    rng = np.random.RandomState(0)
    for _ in range(500):
        i1, j1 = int(rng.randint(-5000, 5000)), int(rng.randint(-5000, 5000))
        i2, j2 = i1 + int(rng.randint(1, 700)), j1 + int(rng.randint(1, 700))
        for scale in (4, 8):
            got = H.padded_window(i1, j1, i2, j2, scale)
            assert got == P.padded_window(i1, j1, i2, j2, scale)
            pi1, pj1, pi2, pj2 = got
            assert pi1 % scale == pj1 % scale == pi2 % scale == pj2 % scale == 0
            assert pi1 <= i1 - 6 * scale and pi2 >= i2 + 6 * scale and pi1 > i1 - 7 * scale - 1
    # torchvision's int-size rule (shorter edge): the cases the goldens exercise
    assert H._resized_output_size(96, 80, 10) == (12, 10)
    assert H._resized_output_size(64, 136, 17) == (17, 36)
    assert H._resized_output_size(128, 128, 16) == (16, 16)


def test_read_out_refuses_cpu_tensors():
    import torch

    from terrain_diffusion_b200 import _lib as L
    from terrain_diffusion_b200.inference import postproc as H
    with pytest.raises(L.TdxError):
        H.resize_bilinear(torch.zeros(8, 8), (16, 16))
    with pytest.raises(L.TdxError):
        H.gaussian_blur(torch.zeros(16, 16), 11, 5.0)


@pytest.mark.parametrize("name", list(ELEV_WINDOWS))
def test_oracle_compute_climate_matches_reference_golden(name):
    """Groundwork for the device version of WorldPipeline._compute_climate (world_pipeline.py:1314-1365): the restated
    lapse-rate regression + border-clamped bilinear grid_sample agree with the reference on all five output channels."""
    i1, j1, i2, j2 = ELEV_WINDOWS[name]
    c = P.compute_climate(i1, j1, i2, j2, G[f"elev_{name}"], coarse_canvas().planes, 8)
    g = G[f"climate_{name}"]                               # stored at every other pixel
    assert c.shape == (5, i2 - i1, j2 - j1)
    for k in range(5):
        assert rel(c[k, ::2, ::2], g[k]) < 2e-6, k
    assert float(c[4].min()) >= -0.012 - 1e-9 and float(c[4].max()) <= 1e-9   # lapse rate stays inside beta_clip


def test_coastal_lapse_rate_takes_every_branch_and_matches_reference_golden():
    """The coastal coarse map runs every branch of local_baseline_temperature_torch (postprocessing.py:262-326) with
    the thresholds _compute_climate passes: all-ocean windows (den = 0), land fractions 4/225 and 5/225 on either side
    of fallback_threshold 0.02, flat land (var_e < 1) and slopes past both ends of beta_clip."""
    T, c0 = coastal_coarse_map()
    e = (np.sign(c0) * np.square(np.maximum(np.float32(0), c0))).astype(np.float32)     # world_pipeline.py:1329
    t_sea, beta = P.local_baseline_temperature(T, e, 15, fallback_threshold=0.02)
    assert rel(t_sea, GC["t_sea"]) < 2e-6 and np.array_equal(beta, GC["beta"])
    F32 = np.float32
    wm = (e > 0).astype(F32)
    count = np.rint(P._avg_pool_valid(wm, 15) * 225).astype(int)
    den = P._avg_pool_valid(wm, 15)

    def wavg(x):
        return (P._avg_pool_valid((x * wm).astype(F32), 15) / (den + F32(1e-6))).astype(F32)

    mu_T, mu_e, mu_e2, mu_eT = wavg(T), wavg(e), wavg(e * e), wavg(e * T)
    var_e = mu_e2 - mu_e ** 2
    raw = (mu_eT - mu_e * mu_T) / (var_e + F32(1e-6))
    valid = (var_e >= 1.0) & (den >= F32(0.02))
    assert (count == 0).sum() >= 10 and (count == 4).any() and (count == 5).any()
    assert ((den < F32(0.02)) & (count > 0)).sum() >= 3                 # sparse land falls back
    assert ((var_e < 1.0) & (den >= F32(0.02))).sum() >= 3              # flat land falls back
    assert (valid & (raw > 0.0)).sum() >= 3 and (valid & (raw < -0.012)).sum() >= 3      # clipped at both ends
    assert ((den < F32(0.02)) | (var_e < 1.0)).sum() == (beta == F32(-0.0065)).sum()
    assert set(np.unique(beta[valid])) <= {F32(0.0), F32(-0.012)}


def test_oracle_coastal_climate_matches_reference_golden():
    i1, j1, i2, j2 = COASTAL_WINDOW
    c = P.compute_climate(i1, j1, i2, j2, coastal_elev(), coastal_canvas().planes, COASTAL_SCALE)
    g = GC["climate"]                                      # stored at every fourth pixel
    assert c.shape == (5, i2 - i1, j2 - j1)
    for k in range(5):
        assert rel(c[k, ::4, ::4], g[k]) < 2e-6, k


def test_oracle_int16_packing_edges():
    """api.py:73-77 (np.clip(np.floor(a), -32768, 32767).astype('<i2')) on x86 at the edges of the clip."""
    a = np.array([np.nan, np.inf, -np.inf, -32768.5, -32769.0, 32767.9, 32768.0, -1e-30, -0.0, 0.0, 2.0 ** 23 + 1,
                  -(2.0 ** 24), 1.5, -1.5], np.float32)
    want = [0, 32767, -32768, -32768, -32768, 32767, 32767, -1, 0, 0, 32767, -32768, 1, -2]
    got = P.elev_to_int16(a)
    assert got.dtype == np.dtype("<i2") and got.tolist() == want


def test_pipeline_get_wires_the_read_out_like_the_reference(monkeypatch):
    """TerrainPipeline.get / get_elev (WorldPipeline.get, world_pipeline.py:1367-1384): canvases, compression factor and
    the residual statistics reach compute_elev / compute_climate; missing statistics and empty windows are errors."""
    from terrain_diffusion_b200.inference import postproc as H
    from terrain_diffusion_b200.inference.pipeline import TerrainPipeline
    calls = {}

    def fake_elev(resid, lat, i1, j1, i2, j2, scale, mean, std, sigma=5, as_int16=False):
        calls["elev"] = (resid, lat, i1, j1, i2, j2, scale, mean, std, as_int16)
        return "ELEV16" if as_int16 else "ELEV"

    def fake_climate(coarse, i1, j1, i2, j2, elev, scale):
        calls["climate"] = (coarse, i1, j1, i2, j2, elev, scale)
        return "CLIMATE"

    monkeypatch.setattr(H, "compute_elev", fake_elev)
    monkeypatch.setattr(H, "compute_climate", fake_climate)
    p = object.__new__(TerrainPipeline)
    p._residual, p._latents, p._coarse, p.lc = "R", "L", "C", 8
    p._host_views = False
    p.residual_mean, p.residual_std = None, None
    with pytest.raises(ValueError):
        p.get_elev(0, 0, 8, 8)
    p.residual_mean, p.residual_std = 0.5, 2.0
    assert p.get(-3, 4, 61, 132) == {"elev": "ELEV", "climate": "CLIMATE"}
    assert calls["elev"] == ("R", "L", -3, 4, 61, 132, 8, 0.5, 2.0, False)
    assert calls["climate"] == ("C", -3, 4, 61, 132, "ELEV", 8)
    assert p.get(0, 0, 8, 8, with_climate=False) == {"elev": "ELEV", "climate": None}
    assert p.get_elev(0, 0, 8, 8, residual_mean=1.0, residual_std=3.0, as_int16=True) == "ELEV16"
    assert calls["elev"][7:] == (1.0, 3.0, True)


def test_pipeline_small_api_mirrors_world_pipeline(monkeypatch):
    """seed / change_seed / set_cond_snr / empty_cache / context manager / native_resolution (world_pipeline.py:293,331,
    690-712,743-779).  The canvases and stage kernels are replaced by recorders so the constructor runs without a GPU."""
    import torch
    from types import SimpleNamespace

    from terrain_diffusion_b200.inference import pipeline as PL
    from terrain_diffusion_b200.inference.noise import next_seed

    class RecCanvas:
        def __init__(self, channels, f, win, dev, args=(), args_windows=(), batch_size=None, cache_limit=None):
            self.f, self.done = f, set()

        def clear_cache(self):
            self.done.clear()

    seen = {}
    monkeypatch.setattr(PL, "LazyCanvas", RecCanvas)
    monkeypatch.setattr(PL, "linear_weight_window", lambda size, dev: torch.zeros(size, size))
    monkeypatch.setattr(PL, "coarse_stage_tile", lambda *a: seen.setdefault("coarse", a))
    dummy = SimpleNamespace(device=torch.device("cpu"))
    smap = torch.arange(5 * 64 * 64, dtype=torch.float32).view(5, 64, 64)
    p = PL.TerrainPipeline(dummy, dummy, dummy, 2 ** 64 + 7, lambda i1, i2, j1, j2: smap[:, :i2 - i1, :j2 - j1],
                           coarse_means=[0.0] * 6,
                           coarse_stds=[1.0] * 6, cond_snr=[0.5, 0.4, 0.3, 0.2, 0.1], histogram_raw=[0.0] * 5,
                           latents_means=[0.0] * 7, latents_stds=[1.0] * 7, residual_mean=0.1, residual_std=1.2)
    assert p.seed == 7 and p.native_resolution == 90.0
    assert p.change_seed(7) is False and p.change_seed(2 ** 64 + 9) is True and p.seed == 9
    p.coarse.done.add((0, 0))
    p.residual.done.add((1, 2))
    assert p.change_seed(None) is True and 0 <= p.seed < 2 ** 64 and not p.coarse.done and not p.residual.done
    with pytest.raises(ValueError):
        p.set_cond_snr([1.0, 2.0])
    p.latents.done.add((0, 0))
    p.set_cond_snr([1, 2, 3, 4, 5])
    assert not p.latents.done and torch.allclose(p._t_cond, torch.atan(torch.tensor([1.0, 2, 3, 4, 5])))
    assert len(p._cond_inputs) == 5 and abs(float(p._cond_inputs[0]) - float(np.log(1.0 / 8.0))) < 1e-6
    # the coarse stage callback picks up the CURRENT seed and conditioning (world_pipeline.py:909-959)
    p.coarse.f((0, 2, -1))
    args = seen["coarse"]
    assert args[2] == p.seed and args[3] == (0, 2, -1) and torch.equal(args[4], smap) and args[5] is p._t_cond
    assert args[6] is p._cond_inputs
    with p as q:
        q.latents_init.done.add((3, 3))
    assert not p.latents_init.done
    # imported rasters overlay the injected conditioning map (set_custom_conditioning_import, world_pipeline.py:781-819)
    p.residual.done.add((5, 5))
    p.set_custom_conditioning_import(2, np.full((3, 4), 7.0, np.float32), 10, -2, default_value=-1.0)
    assert not p.residual.done                                         # rebuild() dropped the cache
    m = p._conditioning_model_input(8, 16, -4, 4)
    assert m.shape == (5, 8, 8) and torch.equal(m[0], smap[0, :8, :8])
    assert float(m[2, 2, 2]) == 7.0 and float(m[2, 4, 5]) == 7.0 and float(m[2, 5, 2]) == -1.0 and float(m[2, 0, 0]) == -1.0
    with pytest.raises(ValueError):
        p.set_custom_conditioning_import(7, np.zeros((2, 2)), 0, 0)
    # portable_rng.next_seed known answers (computed with the reference: parents 1, 42, 2^63+12345, 2^64-1)
    assert [next_seed(s) for s in (1, 42, 2 ** 63 + 12345, 0xFFFFFFFFFFFFFFFF)] == [
        14210067475669473140, 1039766031909981117, 1104045458667958325, 13583675427266712300]
