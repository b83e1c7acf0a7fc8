"""The synthetic conditioning map without a GPU: the numpy oracle (oracle/synthetic_map.py) against the golden recorded
from the reference's own factory and pipeline methods (tests/golden/synthetic_golden.npz), properties of the oracle's
Perlin restatement, and the host side of inference/synthetic_map.py and of the pipelines' `synthetic_map_stats=`."""
from __future__ import annotations

import json
import random
from pathlib import Path

import numpy as np
import pytest

from oracle import synthetic_map as O
from terrain_diffusion_b200.inference import synthetic_map as S
from terrain_diffusion_b200.inference.pipeline import WorldPipeline
from tests._synthetic_inputs import (CASES, IMPORT_CASES, knot_noise, knot_raw, stand_in_fields, stats_fixture,
                                     stats_mapping, write_stats)

G = np.load(Path(__file__).resolve().parent / "golden" / "synthetic_golden.npz")


def oracle_factory(case: str, noise_fn=stand_in_fields) -> O.Factory:
    seed, draw, fm, _ = CASES[case]
    random.seed(draw)
    return O.Factory(stats_mapping(), fm, seed, noise_fn=noise_fn)


def same_bits(a, b) -> bool:
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    nan = np.isnan(a)
    return bool(np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint8), b[~nan].view(np.uint8)))


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reproduces_factory_golden(case):
    f = oracle_factory(case)
    win = CASES[case][3]
    assert same_bits(f.sample_raw(*win), G[f"case.{case}.raw"])
    assert same_bits(f(*win), G[f"case.{case}.map"])


@pytest.mark.parametrize("case", list(IMPORT_CASES))
def test_oracle_reproduces_import_golden(case):
    win, fcase, imports = IMPORT_CASES[case]
    ci0, ci1, cj0, cj1 = win
    assert same_bits(oracle_factory(fcase)(cj0, ci0, cj1, ci1), G[f"import.{case}.plain"])
    got = O.import_conditioning(oracle_factory(fcase), imports, *win)
    assert same_bits(got, G[f"import.{case}"])
    assert np.isnan(got).any() or case in ("defaults", "big")


def test_oracle_reproduces_knot_golden():
    stats = stats_mapping()
    noise = knot_noise()
    raw = np.stack([O.transform(noise[k], stats[f"noise_quantiles_{k}"], stats[f"base_image_quantiles_{k}"])
                    for k in range(5)])
    assert same_bits(raw, G["knots.raw"])
    assert same_bits(O.finalize(knot_raw(), stats), G["knots.finalize"])
    # the knot noise covers every branch of np.interp: below, above, on the end knots and on inner knots
    for k in range(5):
        xp = stats[f"noise_quantiles_{k}"]
        x = noise[k].ravel().astype(np.float64)
        assert (x < xp[0]).any() and (x > xp[-1]).any() and (x == xp[-1]).any()
        assert np.isin(x, xp[1:-1]).sum() >= 30


def test_non_square_windows_are_the_reference_reinterpretation():
    f = oracle_factory("wide")
    i1, j1, i2, j2 = CASES["wide"][3]
    raw = f.sample_raw(i1, j1, i2, j2)
    xx, yy = np.meshgrid(np.arange(i1, i2, dtype=np.float32), np.arange(j1, j2, dtype=np.float32))
    flat = O.transform(stand_in_fields(f.seeds[0], *f.configs[0], xx, yy).ravel(), f.stats["noise_quantiles_0"],
                       f.stats["base_image_quantiles_0"])
    assert raw.shape[1:] == (i2 - i1, j2 - j1) and np.array_equal(raw[0].ravel(), flat)
    assert not np.array_equal(raw[0], flat.reshape(j2 - j1, i2 - i1).T)


# ------------------------------------------------------------------------------------------------ Perlin properties
@pytest.mark.parametrize("seed", [0, 1337, -5, (1 << 31) - 1])
def test_perlin_is_zero_on_the_lattice_at_one_octave(seed):
    v = O.fbm_plane(seed, 1.0, 1, 2.0, 0.5, -40, -17, 50, 60)
    assert not np.any(v)
    assert np.any(O.fbm_plane(seed, 0.37, 1, 2.0, 0.5, -40, -17, 50, 60))


@pytest.mark.parametrize("octaves,gain", [(1, 0.5), (2, 0.5), (4, 0.5), (5, 0.5), (3, 0.6), (2, 0.6)])
def test_fbm_stays_within_unit_range(octaves, gain):
    v = O.fbm_plane(98765, 0.173, octaves, 2.0, gain, -300, 250, 300, 300)
    assert np.abs(v).max() <= 1.0 and v.std() > 0.05


def test_seed_wraps_as_int32():
    a = O.fbm_plane((1 << 31) - 1, 0.07, 3, 2.0, 0.5, -20, 30, 40, 40)
    # a seed above 2^31 is the same C int as its value minus 2^32
    assert np.array_equal(a, O.fbm_plane((1 << 31) - 1 - (1 << 32), 0.07, 3, 2.0, 0.5, -20, 30, 40, 40))
    # the second octave runs at seed -2^31 (seed++ wraps): rebuild the sum from single octaves
    xx, yy = np.meshgrid(np.arange(30, 70, dtype=np.float32), np.arange(-20, 20, dtype=np.float32))
    x, y = xx * np.float32(0.07), yy * np.float32(0.07)
    amp = O.fractal_bounding(3, 0.5)
    total = np.zeros_like(x)
    for s in ((1 << 31) - 1, -(1 << 31), -(1 << 31) + 1):
        total = total + O.single_perlin(np.int32(s), x, y) * amp
        x, y, amp = x * np.float32(2), y * np.float32(2), np.float32(amp * np.float32(0.5))
    assert np.array_equal(a, total)


def test_gradient_table_is_fastnoiselite_layout():
    g = O.GRADIENTS_2D.reshape(128, 2)
    assert g.dtype == np.float32 and np.array_equal(g[:24], g[24:48]) and np.array_equal(g[120:], g[:8])
    assert np.allclose(np.hypot(g[:, 0], g[:, 1]), 1.0, atol=1e-6)
    assert np.float32(0.130526192220052) == g[0, 0] and np.float32(0.99144486137381) == g[0, 1]


# ------------------------------------------------------------------------------------------------ statistics
def test_stats_from_path_mapping_and_cache(tmp_path, monkeypatch):
    path = tmp_path / "stats.json"
    write_stats(path)
    want = stats_mapping()
    for src in (path, str(path), want):
        got = S.load_stats(src)
        assert set(got) == set(want)
        for k, v in want.items():
            assert np.array_equal(got[k], v)
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError) as e:
        S.load_stats(None)
    assert S.STATS_CACHE_PATH in str(e.value) and "stats=" in str(e.value)
    (tmp_path / "data" / "global").mkdir(parents=True)
    write_stats(tmp_path / S.STATS_CACHE_PATH)
    assert np.array_equal(S.load_stats(None)["noise_quantiles_3"], want["noise_quantiles_3"])
    with pytest.raises(FileNotFoundError, match="stats="):
        S.make_synthetic_map_factory(stats=tmp_path / "missing.json")


def _broken(**change):
    payload = stats_fixture()
    payload.update(change)
    return payload


@pytest.mark.parametrize("what", ["length", "decreasing", "flat", "nan", "short", "missing"])
def test_stats_errors(tmp_path, what):
    payload = stats_fixture()
    noise = [list(t) for t in payload["noise_quantile_tables"]]
    data = [list(t) for t in payload["data_quantile_tables"]]
    if what == "length":
        data[2] = data[2][:-1]
    elif what == "decreasing":
        noise[1][10], noise[1][11] = noise[1][11], noise[1][10]
    elif what == "flat":
        noise[4][20] = noise[4][21]
    elif what == "nan":
        data[0][5] = float("nan")
    elif what == "short":
        noise, data = [t[:1] for t in noise], [t[:1] for t in data]
    payload.update(noise_quantile_tables=noise, data_quantile_tables=data)
    if what == "missing":
        del payload["temp_std_p99"]
    path = tmp_path / "s.json"
    path.write_text(json.dumps(payload))
    with pytest.raises((ValueError, KeyError)):
        S.load_stats(path)
    mapping = stats_mapping(payload) if what != "missing" else {k: v for k, v in stats_mapping().items()
                                                                if k != "temp_std_p99"}
    with pytest.raises(ValueError):
        S.load_stats(mapping)


def test_length_mismatch_message_is_transform_perlins():
    m = stats_mapping()
    m["base_image_quantiles_0"] = m["base_image_quantiles_0"][:10]
    with pytest.raises(ValueError, match="same length"):
        S.make_synthetic_map_factory(stats=m)


@pytest.mark.parametrize("seed", [0, None, 1, 12345, (1 << 31) - 1, 1 << 31, (1 << 32) + 77, (1 << 64) - 1])
def test_seed_derivation(seed):
    random.seed(99)
    want = O.noise_seeds(seed)
    random.seed(99)
    f = S.make_synthetic_map_factory(seed=seed, stats=stats_mapping())
    assert f.seeds == want and all(0 <= s < (1 << 31) for s in f.seeds)
    if seed:
        assert want == [(seed + k + 1) & 0x7FFFFFFF for k in range(5)]


# ------------------------------------------------------------------------------------------------ pipeline keyword
def test_pipeline_keyword_checks(tmp_path):
    m = stats_mapping()
    with pytest.raises(ValueError, match="not both"):
        WorldPipeline(seed=1, conditioning_fn=lambda *a: None, synthetic_map_stats=m)
    with pytest.raises(FileNotFoundError):
        WorldPipeline(seed=1, synthetic_map_stats=tmp_path / "nope.json")
    with pytest.raises(ValueError):
        WorldPipeline(seed=1, synthetic_map_stats={"a_temp_std": 1.0})
    with pytest.raises(ValueError):
        WorldPipeline(seed=1, synthetic_map_stats=m, frequency_mult=[1.0, 2.0])
    p = WorldPipeline(seed=(1 << 64) - 1, synthetic_map_stats=m)
    assert p._synthetic.seeds == O.noise_seeds((1 << 64) - 1)
    assert p._synthetic.frequency_mult == [1.5, 3.0, 3.0, 3.0, 3.0]
    # never written into config.json: a path there would be a host path
    p.save_pretrained(tmp_path / "saved")
    cfg = json.loads((tmp_path / "saved" / "config.json").read_text())
    assert "synthetic_map_stats" not in cfg and cfg["frequency_mult"] == [1.5, 3, 3, 3, 3]
    # seeds follow change_seed and rebuild, as the reference's _init_conditioning re-derives them
    assert p.change_seed(4242) and p._synthetic.seeds == O.noise_seeds(4242)
    p.seed = 777
    p.rebuild()
    assert p._synthetic.seeds == O.noise_seeds(777)
    q = WorldPipeline(seed=5, synthetic_map_stats=m, frequency_mult=[1, 1, 1, 1, 2])
    assert q._synthetic.frequency_mult == [1.0, 1.0, 1.0, 1.0, 2.0]
    assert WorldPipeline(seed=5)._synthetic is None


def test_device_is_required():
    f = S.make_synthetic_map_factory(seed=3, stats=stats_mapping(), device=None)
    with pytest.raises(Exception):
        S.make_synthetic_map_factory(seed=3, stats=stats_mapping(), device="cpu")
    with pytest.raises(ValueError):
        f(0, 0, 0, 5)
    with pytest.raises(ValueError):
        f(0, 0, 1.5, 5)
