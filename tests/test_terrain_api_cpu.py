"""Terrain API read-out, CPU side: the oracle restatement of torch's two CPU bilinear kernels (oracle/terrain_api.py
`upsample_crop`, `terrain_payload`) against the golden vectors recorded from the reference's own `_get_terrain` /
`_binary_response` (tests/golden/make_golden_terrain_api.py) and against live torch, the argument checks, and the
wiring of `WorldPipeline.get_terrain` / `terrain_payload` with the device work stubbed out."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import terrain_api as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import postproc as P
from tests._terrain_api_inputs import CASES, case_world, planes

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "terrain_api_golden.npz")


def same_bits(got, want):
    """Bit-identical except that NaN only has to be NaN (its sign and payload are the producer's)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(want)
    return (got.shape == want.shape and np.array_equal(np.isnan(got), nan)
            and np.array_equal(got.view(np.uint32)[~nan], want.view(np.uint32)[~nan]))


def oracle_case(name):
    world, (i1, j1, i2, j2, scale) = case_world(name)
    ni1, nj1, ni2, nj2, oi, oj = O.terrain_window(i1, j1, i2, j2, scale)
    native = planes(world.seed, ni1, nj1, ni2, nj2, world.specials)
    with np.errstate(invalid="ignore"):
        up = O.upsample_crop(native, scale, oi, oj, i2 - i1, j2 - j1)
    return up[0], up[1:]


def test_golden_records_its_torch():
    assert str(G["torch_version"]).startswith("2.") and str(G["cpu_capability"]) in ("AVX512", "AVX2", "DEFAULT")


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(name):
    elev, climate = oracle_case(name)
    assert same_bits(elev, G[f"{name}.elev"]) and same_bits(climate, G[f"{name}.climate"])
    body = O.terrain_payload(elev, climate)
    assert body == G[f"{name}.body"].tobytes()
    assert tuple(G[f"{name}.hw"]) == elev.shape


def test_golden_cases_take_both_torch_paths():
    paths = {}
    for name, (_, _, i1, j1, i2, j2, scale) in CASES.items():
        ni1, nj1, ni2, nj2, _, _ = O.terrain_window(i1, j1, i2, j2, scale)
        if scale > 1:
            paths[name] = ((ni2 - ni1) + (nj2 - nj1)) * scale
    assert paths["s2_edge128"] == 128 and paths["s2_edge130"] == 130
    assert sum(v <= 128 for v in paths.values()) >= 5 and sum(v > 128 for v in paths.values()) >= 5
    assert any(np.isnan(G[f"{n}.elev"]).any() for n in CASES if n.startswith("specials"))
    e = np.concatenate([G[f"{n}.elev"].ravel() for n in CASES])
    assert (e > 32767).any() and (e < -32768).any()           # both int16 clip edges are packed


@pytest.mark.parametrize("scale", [2, 3, 5, 8, 16])
def test_oracle_matches_live_torch(scale):
    """Both kernels of this host's torch on native windows 3..24 and 64..80 wide (either axis), every crop offset."""
    rng = np.random.RandomState(scale)
    shapes = [(3, 3), (3, 24), (24, 3), (7, 13), (3, 64), (64, 3), (9, 80), (17, 17)]
    for h, w in shapes:
        x = (rng.randn(5, h, w) * 400).astype(np.float32)
        x[0, h // 2, w // 2] = np.inf
        x[1, 0, w - 1] = -np.inf
        x[2, h - 1, 0] = np.nan
        full = F.interpolate(torch.from_numpy(x)[None], scale_factor=scale, mode="bilinear",
                             align_corners=False)[0].numpy()
        for oi in range(scale):
            oj = scale - 1 - oi
            H, W = h * scale - oi - rng.randint(0, scale), w * scale - oj - rng.randint(0, scale)
            with np.errstate(invalid="ignore"):
                got = O.upsample_crop(x, scale, oi, oj, H, W)
            assert same_bits(got, full[:, oi:oi + H, oj:oj + W]), (h, w, scale, oi, oj)


def test_terrain_window_is_the_reference_arithmetic():
    rng = np.random.RandomState(0)
    for _ in range(500):
        scale = int(rng.choice([1, 2, 3, 4, 7, 8, 16]))
        i1, j1 = int(rng.randint(-5000, 5000)), int(rng.randint(-5000, 5000))
        i2, j2 = i1 + int(rng.randint(1, 300)), j1 + int(rng.randint(1, 300))
        want = O.terrain_window(i1, j1, i2, j2, scale)
        assert P.terrain_window(i1, j1, i2, j2, scale) == want
        if scale > 1:                                       # api.py:120-153 literally
            ni1, nj1 = i1 // scale, j1 // scale
            assert want[:4] == (ni1 - 1, nj1 - 1, -(-i2 // scale) + 1, -(-j2 // scale) + 1)
            assert want[4:] == (scale + i1 - ni1 * scale, scale + j1 - nj1 * scale)
            assert 0 <= want[4] - scale < scale and want[4] + (i2 - i1) <= (want[2] - want[0]) * scale


def _no_device(*a, **k):
    raise AssertionError("device work before the argument checks")


def test_argument_errors_come_before_any_device_work(monkeypatch):
    from terrain_diffusion_b200.inference.pipeline import WorldPipeline
    monkeypatch.setattr(L, "lib", _no_device)
    monkeypatch.setattr(P, "upsample_crop", _no_device)
    p = WorldPipeline()
    p._get_device = _no_device
    bad = [(0, 0, 4, 4, 0), (0, 0, 4, 4, -2), (0, 0, 4, 4, 2.0), (0, 0, 4, 4, True), (0, 0, 4, 4, "2"),
           (4, 0, 4, 4, 1), (0, 4, 4, 4, 1), (5, 0, 4, 4, 2), (0, 5, 4, 4, 8), (0.5, 0, 4, 4, 1),
           (0, 0, 70000, 4, 1)]
    for args in bad:
        with pytest.raises(ValueError):
            p.get_terrain(*args)
        with pytest.raises(ValueError):
            p.terrain_payload(*args)


def test_get_terrain_and_payload_wiring(monkeypatch):
    from terrain_diffusion_b200.inference.pipeline import WorldPipeline
    calls = []

    def fake_upsample(elev, climate, scale, oi, oj, H, W, payload=False):
        calls.append(("up", tuple(elev.shape), None if climate is None else tuple(climate.shape), scale, oi, oj, H, W,
                      payload))
        return torch.arange(H * W * 18, dtype=torch.uint8) if payload else torch.zeros(6 if climate is not None else 1,
                                                                                        H, W)

    monkeypatch.setattr(P, "upsample_crop", fake_upsample)
    monkeypatch.setattr(P, "to_host", lambda t: calls.append(("host",)) or t)
    p = WorldPipeline()

    def fake_device(i1, j1, i2, j2, with_climate=True):
        calls.append(("get", i1, j1, i2, j2, with_climate))
        return {"elev": torch.zeros(i2 - i1, j2 - j1),
                "climate": torch.zeros(5, i2 - i1, j2 - j1) if with_climate else None}

    p._get_device = fake_device
    out = p.get_terrain(-13, 29, 3, 45, scale=8)
    assert calls == [("get", -3, 2, 2, 7, True), ("up", (5, 5), (5, 5, 5), 8, 11, 13, 16, 16, False), ("host",)]
    assert tuple(out["elev"].shape) == (16, 16) and tuple(out["climate"].shape) == (5, 16, 16)
    calls.clear()
    out = p.get_terrain(-7, -7, 5, 2, scale=1, with_climate=False)    # scale 1: the window itself, no padding
    assert calls == [("get", -7, -7, 5, 2, False), ("up", (12, 9), None, 1, 0, 0, 12, 9, False), ("host",)]
    assert out["climate"] is None and tuple(out["elev"].shape) == (12, 9)
    calls.clear()
    body, hw = p.terrain_payload(-1, -1, 2, 3, scale=2)
    assert hw == (3, 4) and body == bytes(range(216))
    assert calls == [("get", -2, -2, 2, 3, True), ("up", (4, 5), (5, 4, 5), 2, 3, 3, 3, 4, True), ("host",)]
    calls.clear()
    p._host_views = False                                          # TerrainPipeline: device tensors, no copy
    p.get_terrain(0, 0, 4, 4, scale=2)
    assert [c[0] for c in calls] == ["get", "up"]


def test_bench_terrain_api_help_runs():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_terrain_api.py"), "--help"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--iters" in out.stdout and "--sizes" in out.stdout and "--scales" in out.stdout
