"""Minecraft API read-out, CPU side: the oracle (oracle/minecraft_api.py, a per-pixel decision list) against the golden
vectors recorded from the reference's own mask-chain classifier (tests/golden/make_golden_minecraft.py), its Sobel
restatement against live torch, the reach of every decision-tree leaf and quirk across the golden cases, the window
arithmetic, the argument errors, the noise-provider calls and the missing-pyfastnoiselite error."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import minecraft_api as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import minecraft as M
from tests._minecraft_inputs import (BODY_LIMIT, CASES, FULL_LIMIT, FastNoiseLite, case_world, digest, install_stand_in,
                                     stand_in_noise)

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "minecraft_golden.npz")


def same_bits(got, want):
    """Bit-identical except that NaN only has to be NaN (its sign and payload are the producer's)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(want)
    return (got.shape == want.shape and np.array_equal(np.isnan(got), nan)
            and np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan]))


def planes_fn(i0, j0, h, w):
    return np.stack([stand_in_noise(c, i0, j0, h, w) for c in M.NOISE_CONFIGS])


def oracle_case(name):
    world, (i1, j1, i2, j2, scale, noise) = case_world(name)
    return O.request(world.get_np, i1, j1, i2, j2, scale, noise, world.native_resolution, planes_fn)


_ORACLE = {}


def cached_case(name):
    if name not in _ORACLE:
        _ORACLE[name] = oracle_case(name)
    return _ORACLE[name]


def test_golden_records_its_torch():
    assert str(G["torch_version"]).startswith("2.") and str(G["cpu_capability"]) in ("AVX512", "AVX2", "DEFAULT")


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(name):
    r = cached_case(name)
    if f"{name}.error" in G:                   # the reference cannot serve a one-column window taller than one row
        H, W = r["elev"].shape
        assert W == 1 and H > 1 and "IndexError" in str(G[f"{name}.error"])
        return
    assert digest(np.frombuffer(r["body"], np.uint8)) == str(G[f"{name}.body.sha256"]), "body"
    if r["elev"].size <= BODY_LIMIT:
        assert r["body"] == G[f"{name}.body"].tobytes(), "body"
    assert tuple(G[f"{name}.hw"]) == r["elev"].shape
    for k in ("elev", "elev_smooth", "climate", "biome"):          # every case: the whole array, by its digest
        assert digest(r[k]) == str(G[f"{name}.{k}.sha256"]), k
    if r["elev"].size <= FULL_LIMIT:                               # small cases: element by element
        assert same_bits(r["elev"], G[f"{name}.elev"]), "elev"
        assert same_bits(r["elev_smooth"], G[f"{name}.elev_smooth"]), "elev_smooth"
        assert same_bits(r["climate"], G[f"{name}.climate"]), "climate"
        assert np.array_equal(r["biome"], G[f"{name}.biome"]), "biome"


def test_digest_sees_every_bit_but_not_nan_payloads():
    a = np.linspace(-3, 3, 12, dtype=np.float32).reshape(3, 4)
    b = a.copy()
    b.view(np.uint32)[1, 2] ^= 1
    assert digest(a) != digest(b) and digest(a) != digest(a.reshape(4, 3)) and digest(a) != digest(a.astype(np.int16))
    n1, n2 = a.copy(), a.copy()
    n1[0, 0], n2.view(np.uint32)[0, 0] = np.nan, 0xFFC00001
    assert digest(n1) == digest(n2) != digest(a)


def test_golden_cases_cover_the_arithmetic_paths():
    """Both bilinear kernels, with the switch taken from the 2-padded window; all three Sobel orders; detail noise on
    and off; both int16 packings of NaN-free land and ocean."""
    small, wide, switch, sobel = set(), set(), [], set()
    for name, (_, _, i1, j1, i2, j2, scale, _) in CASES.items():
        wi1, wj1, wi2, wj2, _, _ = O.minecraft_window(i1, j1, i2, j2, scale)
        H, W = i2 - i1, j2 - j1
        if scale > 1:
            h, w = wi2 - wi1, wj2 - wj1
            (small if (h + w) * scale <= 128 else wide).add(name)
            if (h + w) * scale > 128 and (h - 2 + w - 2) * scale <= 128:
                switch.append(name)
        sobel.add("oneDNN" if (H + 2) * (W + 2) > 20480 else "one" if H * W == 1 else
                  "gemm+tail" if (H * W) % 16 else "gemm")
    assert len(small) >= 4 and len(wide) >= 4 and set(switch) >= {"s2_switch", "s4_switch"}
    assert sobel == {"oneDNN", "one", "gemm", "gemm+tail"}
    assert {CASES[n][7] for n in CASES} == {-1.0, 0.0, 1.0} and {CASES[n][1] for n in CASES} == {30.0, 90.0}


@pytest.mark.parametrize("shape", [(3, 3), (3, 4), (4, 3), (3, 40), (40, 3), (6, 6), (18, 18), (18, 40), (50, 51),
                                   (143, 143), (144, 144), (160, 128), (161, 128), (3, 6826), (3, 6827), (202, 302)])
def test_sobel_restatement_matches_live_torch(shape):
    """oracle.sobel against this host's torch conv2d on both sides of its 20480-element dispatch and of the 16-pixel
    gemm blocks, on values whose magnitudes differ widely (so every summation order shows)."""
    rng = np.random.default_rng(sum(shape))
    x = (rng.standard_normal(shape) * 10.0 ** rng.integers(-3, 4, shape)).astype(np.float32)
    sx = torch.tensor([[-1, 0, 1], [-2, 0, 2], [-1, 0, 1]], dtype=torch.float32).view(1, 1, 3, 3) / 8.0
    sy = torch.tensor([[-1, -2, -1], [0, 0, 0], [1, 2, 1]], dtype=torch.float32).view(1, 1, 3, 3) / 8.0
    t = torch.from_numpy(x)[None, None]
    dx, dy = O.sobel(x)
    assert np.array_equal(dx, torch.nn.functional.conv2d(t, sx)[0, 0].numpy())
    assert np.array_equal(dy, torch.nn.functional.conv2d(t, sy)[0, 0].numpy())


# Quirks of the mask chain that the decision list must reproduce, counted over the golden cases.
MIN_LEAF_PIXELS = 10
MIN_QUIRK_PIXELS = 5


def test_every_leaf_and_quirk_is_reached():
    counts = np.zeros(len(O.LEAVES), np.int64)
    quirks = dict.fromkeys(("desert_then_grove", "warm_sparse_demoted_plains", "bare_override_above_lowland",
                            "bare_override_midland_or_lowland", "steep_ocean_floor_kept", "nan_temp_land_plains",
                            "nan_temp_ocean_44"), 0)
    for name in CASES:
        r = cached_case(name)
        leaf, v = r["leaf"], r["vars"]
        counts += np.bincount(leaf.ravel(), minlength=len(O.LEAVES))
        t = v["temp"]
        name_of = np.array(O.LEAF_NAMES)[leaf]
        quirks["desert_then_grove"] += int(((name_of == "dry_steppe") & (t >= 20.0)).sum())
        quirks["warm_sparse_demoted_plains"] += int((name_of == "sf_warm_demoted").sum())
        bare = (name_of == "bare") | (name_of == "bare_snow")
        quirks["bare_override_above_lowland"] += int((bare & ~v["lowland"] & ~v["mountains"]).sum())
        quirks["bare_override_midland_or_lowland"] += int((bare & ~v["mountains"]).sum())
        quirks["steep_ocean_floor_kept"] += int((v["ocean"] & v["slope_bare"]).sum())
        quirks["nan_temp_land_plains"] += int((np.isnan(t) & ~v["ocean"] & (r["biome"] == 1)).sum())
        quirks["nan_temp_ocean_44"] += int((np.isnan(t) & v["ocean"] & (r["biome"] == 44)).sum())
        assert not (np.isnan(t) & ~v["ocean"] & (r["biome"] != 1) & ~v["slope_bare"]).any()
        assert not (np.isnan(t) & v["ocean"] & (r["biome"] != 44)).any()
    low = {n: int(c) for n, c in zip(O.LEAF_NAMES, counts) if c < MIN_LEAF_PIXELS}
    assert not low, f"leaves reached by fewer than {MIN_LEAF_PIXELS} pixels: {low}"
    few = {k: c for k, c in quirks.items() if c < MIN_QUIRK_PIXELS}
    assert not few, f"quirks reached by fewer than {MIN_QUIRK_PIXELS} pixels: {few}"
    print("\nleaf pixels:", dict(zip(O.LEAF_NAMES, counts.tolist())), "\nquirk pixels:", quirks)


def test_window_arithmetic_is_the_reference():
    rng = np.random.RandomState(0)
    for _ in range(500):
        scale = int(rng.choice([1, 2, 3, 4, 7, 8, 16]))
        i1, j1 = int(rng.randint(-5000, 5000)), int(rng.randint(-5000, 5000))
        i2, j2 = i1 + int(rng.randint(1, 300)), j1 + int(rng.randint(1, 300))
        got = M.minecraft_window(i1, j1, i2, j2, scale)
        assert got == O.minecraft_window(i1, j1, i2, j2, scale)
        if scale > 1:                                        # minecraft_api.py:273-303 literally
            ni1, nj1 = i1 // scale, j1 // scale
            assert got[:4] == (ni1 - 2, nj1 - 2, -(-i2 // scale) + 2, -(-j2 // scale) + 2)
            assert got[4:] == (2 * scale + i1 - ni1 * scale, 2 * scale + j1 - nj1 * scale)
            h, w = got[2] - got[0], got[3] - got[1]
            assert got[4] >= 1 and got[4] + (i2 - i1) + 1 <= h * scale and got[5] + (j2 - j1) + 1 <= w * scale
        else:
            assert got == (i1 - 1, j1 - 1, i2 + 1, j2 + 1, 1, 1)


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


def test_argument_errors_come_before_any_device_work(monkeypatch):
    from terrain_diffusion_b200.inference.pipeline import WorldPipeline
    monkeypatch.setattr(L, "lib", _no_device)
    monkeypatch.setattr(M, "readout", _no_device)
    p = WorldPipeline()
    p._get_device = _no_device
    bad = [((0, 0, 4, 4, 0), {}), ((0, 0, 4, 4, -2), {}), ((0, 0, 4, 4, 2.0), {}), ((0, 0, 4, 4, True), {}),
           ((0, 0, 4, 4, "2"), {}), ((4, 0, 4, 4, 1), {}), ((0, 4, 4, 4, 1), {}), ((5, 0, 4, 4, 2), {}),
           ((0, 5, 4, 4, 8), {}), ((0.5, 0, 4, 4, 1), {}), ((0, 0, 70000, 4, 1), {}), ((0, 0, 4, 4, 2), {"noise": "1"}),
           ((0, 0, 4, 4, 2), {"noise": None}), ((0, 0, 4, 4, 2), {"noise": True})]
    for args, kw in bad:
        with pytest.raises(ValueError):
            p.get_minecraft(*args, noise_fn=_no_device, **kw)
        with pytest.raises(ValueError):
            p.minecraft_payload(*args, noise_fn=_no_device, **kw)


def _wired_pipeline(monkeypatch, calls):
    from terrain_diffusion_b200.inference import postproc as P
    from terrain_diffusion_b200.inference.pipeline import WorldPipeline

    def fake_readout(elev, climate, noise, scale, oi, oj, H, W, noise_scale, psm, nr, centre=None, payload=False):
        calls.append(("readout", tuple(elev.shape), None if climate is None else tuple(climate.shape),
                      None if centre is None else tuple(centre.shape), scale, oi, oj, H, W, noise_scale, psm, nr,
                      payload))
        if payload:
            return torch.arange(4 * H * W, dtype=torch.uint8)
        return torch.zeros(7 if climate is not None else 2, H, W), torch.ones(H, W, dtype=torch.int16)

    monkeypatch.setattr(M, "readout", fake_readout)
    monkeypatch.setattr(P, "to_host", lambda t: calls.append(("host",)) or t)
    p = WorldPipeline(native_resolution=30.0)

    def fake_device(i1, j1, i2, j2, with_climate=True):
        calls.append(("get", i1, j1, i2, j2, with_climate))
        return {"elev": torch.zeros(i2 - i1, j2 - j1),
                "climate": torch.zeros(5, i2 - i1, j2 - j1) if with_climate else None}

    p._get_device = fake_device
    return p


def test_pipeline_wiring_and_one_provider_call_per_configuration(monkeypatch):
    calls, seen = [], []

    def noise_fn(cfg, i0, j0, h, w):
        seen.append((cfg, i0, j0, h, w))
        return np.full((h, w), 0.5, np.float32)

    p = _wired_pipeline(monkeypatch, calls)
    out = p.get_minecraft(-13, 29, 3, 45, scale=8, noise=0.5, noise_fn=noise_fn)
    assert calls == [("get", -4, 1, 3, 8, True), ("readout", (7, 7), (5, 7, 7), None, 8, 19, 21, 16, 16, 0.5, 3.75,
                                                    30.0, False), ("host",), ("host",)]
    assert sorted(seen) == sorted((c, -13, 29, 16, 16) for c in M.NOISE_CONFIGS)   # five configurations, once each
    assert tuple(out["elev"].shape) == (16, 16) and tuple(out["climate"].shape) == (5, 16, 16)
    assert out["biome"].dtype == torch.int16
    calls.clear(), seen.clear()
    body, hw = p.minecraft_payload(-7, -7, 5, 2, scale=1, noise=1.0, noise_fn=noise_fn)   # scale 1: two reads
    assert hw == (12, 9) and body == bytes(range(256)) * (432 // 256) + bytes(range(432 % 256))
    assert calls == [("get", -8, -8, 6, 3, False), ("get", -7, -7, 5, 2, True),
                     ("readout", (14, 11), (5, 12, 9), (12, 9), 1, 1, 1, 12, 9, 1.0, 30.0, 30.0, True), ("host",)]
    assert sorted(seen) == sorted((c, -7, -7, 12, 9) for c in (M.TEMP_COARSE, M.TEMP_FINE, M.PRECIP))
    calls.clear(), seen.clear()
    p.get_minecraft(0, 0, 4, 4, scale=2, noise=0, noise_fn=noise_fn)      # no detail noise: three configurations
    assert len(seen) == 3 and {s[0] for s in seen} == {M.TEMP_COARSE, M.TEMP_FINE, M.PRECIP}
    calls.clear()
    p._host_views = False                                                  # TerrainPipeline: device tensors, no copy
    p.get_minecraft(0, 0, 4, 4, scale=2, noise_fn=noise_fn)
    assert [c[0] for c in calls] == ["get", "readout"]


def test_noise_provider_shape_is_checked(monkeypatch):
    p = _wired_pipeline(monkeypatch, [])
    with pytest.raises(ValueError, match="noise_fn returned shape"):
        p.get_minecraft(0, 0, 4, 4, scale=2, noise_fn=lambda cfg, i0, j0, h, w: np.zeros((w, h + 1), np.float32))


def test_five_configurations_are_the_references_seven_generators():
    """_TEMP_NOISE == _SNOW_NOISE and _TEMP_NOISE_FINE == _SNOW_NOISE_FINE (minecraft_api.py:127-186)."""
    assert len(set(M.NOISE_CONFIGS)) == 5
    assert M.TEMP_COARSE == (12345, 1 / 500, 3, 2.0, 0.5) and M.TEMP_FINE == (54321, 1 / 128, 2, 2.0, 0.5)
    assert M.PRECIP == (12345, 1 / 500, 5, 2.0, 0.5)
    assert M.ELEV_COARSE == (99999, 1 / 24, 3, 2.0, 0.5) and M.ELEV_FINE == (88888, 1 / 6, 2, 2.0, 0.6)


def test_default_provider_needs_pyfastnoiselite(monkeypatch):
    M._generator.cache_clear()
    monkeypatch.setitem(sys.modules, "pyfastnoiselite", None)
    monkeypatch.setitem(sys.modules, "pyfastnoiselite.pyfastnoiselite", None)
    with pytest.raises(RuntimeError, match=r"noise_fn=\.\.\..*pyfastnoiselite"):
        M.fastnoiselite_noise(M.TEMP_COARSE, 0, 0, 2, 2)
    M._generator.cache_clear()


def test_default_provider_builds_the_reference_generators(monkeypatch):
    """With a module importable as pyfastnoiselite.pyfastnoiselite, the default provider configures it as the reference
    does and samples x = j0 + c, y = i0 + r."""
    M._generator.cache_clear()
    saved = {k: sys.modules.get(k) for k in ("pyfastnoiselite", "pyfastnoiselite.pyfastnoiselite")}
    try:
        install_stand_in()
        for cfg in M.NOISE_CONFIGS:
            got = M.fastnoiselite_noise(cfg, -7, 12, 5, 9)
            assert got.dtype == np.float32 and np.array_equal(got, stand_in_noise(cfg, -7, 12, 5, 9))
        g = M._generator(M.ELEV_FINE)
        assert isinstance(g, FastNoiseLite) and g.frequency == 1 / 6 and g.fractal_gain == 0.6
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        M._generator.cache_clear()


def test_stand_in_depends_on_every_configuration_field():
    base = M.TEMP_COARSE
    ref = stand_in_noise(base, 3, 4, 6, 7)
    assert np.array_equal(ref, stand_in_noise(base, 3, 4, 6, 7)) and np.abs(ref).max() <= 1.0
    for k in range(5):
        changed = list(base)
        changed[k] = changed[k] + (1 if k in (0, 2) else 0.25 if k != 1 else 1 / 1000)
        assert not np.array_equal(ref, stand_in_noise(M.NoiseConfig(*changed), 3, 4, 6, 7)), base._fields[k]


def test_bench_minecraft_api_help_runs():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_minecraft_api.py"), "--help"],
                         capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--iters" in out.stdout and "--sizes" in out.stdout and "--scales" in out.stdout
