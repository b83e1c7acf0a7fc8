"""The explorer's coarse map and the random sampler's land search, CPU side: the oracle restatement
(oracle/coarse_view.py) against the golden vectors recorded from the reference's own functions
(tests/golden/make_golden_coarse_view.py), the argument checks, the `lut=` / missing-matplotlib rule and the wiring of
`WorldPipeline.get_coarse / coarse_image / coarse_data / coarse_stats / land_tiles` and the sampler drop-ins."""
import random
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import coarse_view as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import coarse_view as CV
from terrain_diffusion_b200.inference.pipeline import WorldPipeline
from tests._coarse_view_inputs import (CLIMATE_CELLS, DATA_CASES, LAND_CASES, LAND_WINDOW, PNG_CASES, SAMPLE_CASES,
                                       seeded_lut, world_sums)

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "coarse_view_golden.npz")
WINDOW = ("ci0", "ci1", "cj0", "cj1")
DEFAULT_WINDOW = {"ci0": -50, "ci1": 50, "cj0": -50, "cj1": 50}


def png_args(args):
    """(window, channel, filters) of a coarse_png request as the handler reads it."""
    win = tuple(args.get(k, DEFAULT_WINDOW[k]) for k in WINDOW)
    filters = {}
    for ch in range(6):
        lo, hi = args.get(f"ch{ch}_min"), args.get(f"ch{ch}_max")
        if lo is not None or hi is not None:
            filters[ch] = (lo, hi)
    return win, args.get("channel", 0), filters


def oracle_png(name):
    kind, args = PNG_CASES[name]
    win, channel, filters = png_args(args)
    planes = O.coarse_planes(world_sums(kind, *win))
    with np.errstate(invalid="ignore", over="ignore"):
        return O.coarse_image(planes, channel, seeded_lut(), filters)


@pytest.mark.parametrize("name", list(PNG_CASES))
def test_oracle_matches_reference_png_golden(name):
    img, vmin, vmax = oracle_png(name)
    assert np.array_equal(img, G[f"png.{name}.image"])
    assert [str(round(vmin, 3)), str(round(vmax, 3))] == G[f"png.{name}.headers"].tolist()


@pytest.mark.parametrize("name", list(DATA_CASES))
def test_oracle_matches_reference_data_and_stats_golden(name):
    kind, win = DATA_CASES[name]
    planes = O.coarse_planes(world_sums(kind, *(win[k] for k in WINDOW)))
    data = O.coarse_data(planes)
    assert data.dtype == np.float32
    assert np.array_equal(data.astype(np.float64), G[f"data.{name}"], equal_nan=True)
    stats = O.coarse_stats(planes)
    got = np.array([[stats[c]["min"], stats[c]["max"]] for c in range(6)])
    assert np.array_equal(got, G[f"stats.{name}"], equal_nan=True)
    assert [stats[c]["name"] for c in range(6)] == O.CHANNEL_NAMES == CV.CHANNEL_NAMES


@pytest.mark.parametrize("cw,detail,frac", LAND_CASES)
def test_oracle_matches_reference_land_golden(cw, detail, frac):
    tiles = O.land_tiles(world_sums("mixed", -cw, cw, -cw, cw), -cw, -cw, detail, frac)
    assert np.array_equal(np.array(tiles, np.int64).reshape(-1, 2), G[f"land.{cw}.{detail}.{frac}"])


@pytest.mark.parametrize("seed,detail,frac,n", SAMPLE_CASES)
def test_sampler_drop_in_matches_reference_pick(seed, detail, frac, n, capsys):
    class World:
        def land_tiles(self, cw, d, f):
            return O.land_tiles(world_sums("mixed", -cw, cw, -cw, cw), -cw, -cw, d, f)

    random.seed(seed)
    pick = CV.sample_land_tiles(World(), LAND_WINDOW, detail, frac, n)
    assert np.array_equal(np.array(pick, np.int64).reshape(-1, 2), G[f"sample.{seed}"])
    found = len(World().land_tiles(LAND_WINDOW, detail, frac))
    warned = f"Warning: Only found {found} valid land tiles (requested {n})" in capsys.readouterr().out
    assert warned == (found < n)


@pytest.mark.parametrize("ci,cj", CLIMATE_CELLS)
def test_climate_info_matches_reference(ci, cj):
    sums = world_sums("nan", ci, ci + 1, cj, cj + 1)
    info = O.climate_info(sums)
    want = G[f"climate.{ci}.{cj}"]
    assert np.array_equal([info["temp"], info["temp_std"], info["precip"], info["precip_cv"]], want, equal_nan=True)

    class World:
        def get_coarse(self, a, b, c, d, eps=True):
            assert (a, b, c, d, eps) == (ci, ci + 1, cj, cj + 1, False)
            return torch.from_numpy(O.coarse_planes(world_sums("nan", a, b, c, d), eps=False))

    got = CV.get_coarse_climate_info(World(), ci, cj)
    assert list(got) == ["temp", "temp_std", "precip", "precip_cv"]
    assert np.array_equal(list(got.values()), want, equal_nan=True)


def test_golden_cases_cover_the_rules():
    assert tuple(int(v) for v in str(G["numpy_version"]).split(".")[:2]) >= (2, 1)
    assert np.array_equal(G["lut"], seeded_lut())
    assert np.all(G["png.all_nan_ch2.image"] == 0) and np.all(G["png.all_nan_ch4.image"] == 0)
    big = G["png.big_ch3.image"]                                    # vmin + 1 == vmin: every cell takes entry 0
    assert np.all(big == big[0, 0]) and big[0, 0, 3] == 255
    assert (G["png.nan_ch0.image"][..., 3] == 0).any() and (G["png.nan_ch0.image"][..., 3] == 255).any()
    assert G["png.flat_ch4.headers"].tolist() == ["4.875", "5.875"]   # log1p(130), then the +1 fix
    # ch1 filters are never read: the image is channel 2's unfiltered one
    assert np.array_equal(G["png.filter_ch1_ignored.image"], G["png.ch2.image"])
    for name in ("filter_lo", "filter_hi", "filter_both", "filter_many", "filter_ch1_and_ch5", "filter_nan"):
        kind, args = PNG_CASES[name]                                # some cells dimmed, some not
        win, channel, _ = png_args(args)
        with np.errstate(invalid="ignore"):
            plain = O.coarse_image(O.coarse_planes(world_sums(kind, *win)), channel, seeded_lut())[0]
        dimmed = (G[f"png.{name}.image"] != plain).any(-1)
        assert 0 < dimmed.sum() < dimmed.size, name
    # the fp32 bound: fp64 comparison would dim the cells whose temperature is exactly 7.25
    planes = O.coarse_planes(world_sums("flat", 0, 21, 0, 19))
    assert (planes[2] == np.float32(7.25)).any() and (planes[2] > np.float32(7.25)).any()
    img = O.coarse_image(planes, 0, seeded_lut(), {2: (None, 7.2499999)})[0]
    assert np.array_equal(img, G["png.filter_fp32_bound.image"])
    mask64 = planes[2].astype(np.float64) <= 7.2499999
    assert not np.array_equal(mask64, O.filter_mask(planes, {2: (None, 7.2499999)}))
    assert len(G["land.24.256.0.0"]) == 0 and len(G["land.24.768.0.0"]) == 46 * 46   # empty window; frac 0 keeps all
    assert 0 < len(G["land.24.1536.0.5"]) < len(G["land.24.1536.0.0"])
    assert np.isinf(G["climate.1.14"]).all() and np.isnan(G["climate.0.0"]).all()


def test_round_is_fp32_multiply_rint_divide():
    x = np.random.RandomState(0).standard_normal(200000).astype(np.float32) * np.float32(1000)
    x[:4] = (0.125, 2.675, -0.005, 1e30)
    want = np.rint(x * np.float32(100)) / np.float32(100)
    assert np.array_equal(O.coarse_data(x[None]), want[None])


def test_range_decoding():
    def key(v):
        b = int(np.array(v, np.float32).view(np.uint32))
        return (~b & 0xFFFFFFFF) if b & 0x80000000 else (b | 0x80000000)

    rng = []
    for lo, hi in [(-3.5, 7.0), (-0.0, 1e-40), (-np.inf, np.inf), (5.0, 5.0), (None, None), (0.0, 0.0), (2.0, 3.0)]:
        rng += [0, 0] if lo is None else [~key(lo) & 0xFFFFFFFF, key(hi)]
    as_int32 = np.array(rng, np.uint32).view(np.int32)
    vals = CV.range_values(as_int32)
    assert vals[0] == (-3.5, 7.0) and vals[2] == (-np.inf, np.inf) and vals[3] == (5.0, 5.0)
    assert np.signbit(vals[1][0]) and vals[1][1] == float(np.float32(1e-40))
    assert all(np.isnan(v) for v in vals[4])
    assert CV.display_range(as_int32, 3) == (5.0, 6.0)             # vmax == vmin: + 1
    assert CV.display_range(as_int32, 4) == (2.0, 3.0)             # channel 4 shows plane 6
    assert CV.display_range(as_int32, 5) == (0.0, 1.0)


def test_filter_bounds():
    bounds, active = CV.filter_bounds({0: (-1.5, None), 1: (3.0, 4.0), 2: (None, 7.2499999), 5: (1e300, -1e300)})
    assert active == (1 << 0) | (1 << 5) | (1 << 10) | (1 << 11)     # ch1 ignored
    assert bounds[0, 0] == -1.5 and bounds[2, 1] == np.float32(7.25)
    assert bounds[5, 0] == np.inf and bounds[5, 1] == -np.inf
    bounds, active = CV.filter_bounds(None)
    assert active == 0 and not bounds.any()


def test_argument_errors_come_before_any_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(L, "lib", no_device)
    p = WorldPipeline(native_resolution=30.0)
    p._coarse_sums = no_device
    lut = seeded_lut()
    for win in [(0, 0, 0, 5), (0, 5, 3, 3), (3, 2, 0, 5), (0, 65536, 0, 4), (0.0, 4, 0, 4), (0, True, 0, 4),
                (0, "4", 0, 4), (0, np.float32(4), 0, 4)]:
        for call in (lambda: p.get_coarse(*win), lambda: p.coarse_image(*win, lut=lut),
                     lambda: p.coarse_data(*win), lambda: p.coarse_stats(*win)):
            with pytest.raises(ValueError):
                call()
    for channel in (-1, 6, 2.0, True, "0", None):
        with pytest.raises(ValueError):
            p.coarse_image(0, 4, 0, 4, channel=channel, lut=lut)
    for filters in ({6: (0, 1)}, {-1: (0, None)}, {0: 5.0}, {0: (1, 2, 3)}, {2: ("1", None)}, {"ch0": (0, 1)}):
        with pytest.raises(ValueError):
            p.coarse_image(0, 4, 0, 4, filters=filters, lut=lut)
    for bad in (np.zeros((255, 3)), np.zeros((256, 4)), np.zeros((256,)), np.zeros((3, 256)),
                np.array([["a"] * 3] * 256)):
        with pytest.raises(ValueError):
            p.coarse_image(0, 4, 0, 4, lut=bad)
    for cw, detail in [(0, 1024), (-3, 1024), (2.0, 1024), (5, -256), (5, 1024.0), (5, True), (40000, 1024)]:
        with pytest.raises(ValueError):
            p.land_tiles(cw, detail, 0.5)


def test_missing_matplotlib_names_lut(monkeypatch):
    monkeypatch.setattr(L, "lib", lambda: (_ for _ in ()).throw(AssertionError("device work")))
    monkeypatch.setitem(sys.modules, "matplotlib", None)           # `import matplotlib` raises ImportError
    monkeypatch.setattr(CV, "_viridis", {})
    p = WorldPipeline(native_resolution=30.0)
    p._coarse_sums = lambda *a: (_ for _ in ()).throw(AssertionError("canvas read"))
    with pytest.raises(RuntimeError, match="lut="):
        p.coarse_image(0, 4, 0, 4)


def test_viridis_is_read_from_matplotlib_once(monkeypatch):
    reads = []

    class Cmap:
        N = 256

        def __call__(self, idx):
            reads.append(1)
            return np.concatenate([seeded_lut()[idx], np.ones((len(idx), 1))], axis=1)

    fake = type(sys)("matplotlib")
    fake.colormaps = {"viridis": Cmap()}
    monkeypatch.setitem(sys.modules, "matplotlib", fake)
    monkeypatch.setattr(CV, "_viridis", {})
    assert np.array_equal(CV.check_lut(None), seeded_lut())
    assert CV.check_lut(None) is CV.check_lut(None) and len(reads) == 1
    assert np.array_equal(CV.check_lut(seeded_lut().astype(np.float32)), seeded_lut().astype(np.float32))


def test_bench_coarse_view_help_runs():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_coarse_view.py"), "--help"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--iters" in out.stdout and "--sizes" in out.stdout
