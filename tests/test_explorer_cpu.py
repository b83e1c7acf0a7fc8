"""The explorer's detail view, CPU side: the oracle restatement (oracle/explorer.py) against the golden vectors recorded
from the reference's own handlers (tests/golden/make_golden_explorer.py), the restated `RdBu_r` table, the argument
checks and the wiring of `WorldPipeline.get_detail` / `detail_raw_payload`."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import explorer as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import explorer as E
from terrain_diffusion_b200.inference import postproc
from terrain_diffusion_b200.inference.pipeline import WorldPipeline
from terrain_diffusion_b200.inference.relief import create_lookup_table
from tests._explorer_inputs import HANDLER_CASES, NATIVE_RESOLUTION, PLANE_CASES, plane_case, world_planes

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "explorer_golden.npz")


def case_window(args):
    return O.detail_window(args.get("ci", 0), args.get("cj", 0), args.get("detail_size", 1024), args.get("pan_i", 0),
                           args.get("pan_j", 0))


@pytest.mark.parametrize("name", list(HANDLER_CASES))
def test_oracle_matches_reference_handler_golden(name):
    kind, endpoint, args = HANDLER_CASES[name]
    window = case_window(args)
    assert window == tuple(int(v) for v in G[f"{name}.window"])
    elev, climate = world_planes(kind, *window)
    H, W = elev.shape
    if endpoint == "raw":
        assert O.detail_raw_body(elev, climate[0]) == G[f"{name}.body"].tobytes()
        assert G[f"{name}.headers"].tolist() == [H, W, 1]
        return
    img = G[f"{name}.image"]
    assert img.dtype == np.uint8 and img.shape == (H, W, 4)
    mode = args.get("mode", "relief")
    if mode in ("elevation", "temperature"):
        assert np.array_equal(O.detail_image(elev, climate[0], mode, NATIVE_RESOLUTION), img)
        return
    ref_rgb = G[f"{name}.relief_rgb"]
    assert np.array_equal(O.relief_rgba(ref_rgb), img)             # the 8-bit step on the reference's own relief
    with np.errstate(invalid="ignore"):
        rgb = O.relief_map(elev, resolution=NATIVE_RESOLUTION)
    assert np.array_equal(np.isnan(rgb), np.isnan(ref_rgb))
    fin = ~np.isnan(ref_rgb)
    assert float(np.abs(rgb[fin] - ref_rgb[fin]).max(initial=0.0)) <= 1e-6


@pytest.mark.parametrize("name", list(PLANE_CASES))
def test_oracle_matches_plane_golden(name):
    plane, cmap = plane_case(name)
    with np.errstate(invalid="ignore", over="ignore"):
        got = O.colour_plane(plane, cmap)
    assert np.array_equal(got, G[f"plane.{name}.image"])


def test_golden_cases_cover_the_rules():
    assert tuple(int(v) for v in str(G["numpy_version"]).split(".")[:2]) >= (2, 1)   # NEP 50 promotion in Normalize
    assert np.all(G["nan_relief.image"][G["nan_relief.image"][..., 3] == 0] == 0)
    assert (G["nan_relief.image"][..., 3] == 0).any() and (G["nan_temperature.image"][..., 3] == 0).any()
    assert np.all(G["plane.all_nan.image"] == 0)                    # NaN range: every pixel the bad colour
    big = G["plane.big_terrain.image"]                              # vmin + 1 == vmin: NaN pixels take colour 0 too
    assert np.all(big == big[0, 0]) and big[0, 0, 3] == 255 and np.isnan(plane_case("big_terrain")[0]).any()
    flat = G["flat_elevation.image"]
    assert np.all(flat == flat[0, 0]) and flat[0, 0, 3] == 255
    # fp64 Normalize steps: fp32 arithmetic throughout would take the neighbouring table entry
    p, _ = plane_case("nep50")
    vmin, vmax = O.nan_range(p)
    fp32 = O.png_rgba(O.colormap((p - np.float32(vmin)) / np.float32(vmax - vmin), "terrain"))
    assert not np.array_equal(fp32, G["plane.nep50.image"])
    assert len(np.unique(G["plane.ramp_rdbu.image"].reshape(-1, 4), axis=0)) == 256
    body = G["raw_specials.body"]
    assert np.frombuffer(body.tobytes(), "<i2", count=12).tolist() == [0, 32767, -32768, 32767, -32768, -1, 0, 32767,
                                                                        -32768, -32768, 0, -1]


def test_rdbu_r_is_the_reversed_segments_not_the_flipped_table():
    lut = E.rdbu_r_lut()
    assert lut.shape == (256, 3) and lut.dtype == np.float64
    assert np.array_equal(lut[0], np.array([0x05, 0x30, 0x61]) / 255)
    assert np.array_equal(lut[255], np.array([0x67, 0x00, 0x1f]) / 255)
    rgb = np.array([[int(h[k:k + 2], 16) / 255 for k in (0, 2, 4)] for h in E.RDBU_HEX])
    vals = np.linspace(0, 1, 11)
    rdbu = np.stack([create_lookup_table(np.column_stack([vals, rgb[:, c], rgb[:, c]])) for c in range(3)], axis=1)
    assert np.abs(rdbu[::-1] - lut).max() < 1e-15
    assert not np.array_equal(rdbu[::-1], lut)                      # 1 - x moves some positions by an ulp


def test_argument_errors_come_before_any_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(L, "lib", no_device)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    p = WorldPipeline(native_resolution=30.0)
    p.get_elev = p._get_device = p._relief_on_device = no_device
    bad = [(0, 0, 0, 5), (0, 0, 5, 0), (3, 0, 2, 5), (0, 0, 65536, 4), (0.0, 0, 4, 4), (0, True, 4, 4),
           (0, 0, "4", 4)]
    for win in bad:
        for mode in ("relief", "elevation", "temperature", "other"):
            with pytest.raises(ValueError):
                p.get_detail(*win, mode=mode)
        with pytest.raises(ValueError):
            p.detail_raw_payload(*win)
    for win in ((0, 0, 1, 8), (0, 0, 8, 1)):                        # the relief needs 2 x 2 (np.gradient)
        with pytest.raises(ValueError):
            p.get_detail(*win)
        with pytest.raises(ValueError):
            p.get_detail(*win, mode="biome")
    with pytest.raises(ValueError):
        E.colour_plane(np.zeros((4, 4), np.float32), "viridis")
    for shape in ((4,), (0, 4), (4, 0), (2, 3, 4)):
        with pytest.raises(ValueError):
            E.colour_plane(np.zeros(shape, np.float32), "terrain")
    with pytest.raises(L.TdxError):                                 # valid arguments, no CUDA device
        E.colour_plane(np.zeros((4, 4), np.float32), "terrain")


def test_get_detail_and_raw_payload_wiring(monkeypatch):
    calls = []
    elev, climate = torch.full((3, 4), 7.0), torch.arange(60.0).reshape(5, 3, 4)
    rgb = torch.zeros(3, 4, 3)

    def get_elev(*win):
        calls.append(("get_elev", win))
        return elev

    def get_device(*a):
        calls.append(("_get_device", a))
        return {"elev": elev, "climate": climate}

    def relief(*win, **kw):
        calls.append(("relief", win, kw))
        return rgb

    monkeypatch.setattr(E, "colour_image", lambda x, cmap: calls.append(("colour", x, cmap)) or torch.ones(3, 4, 4))
    monkeypatch.setattr(E, "relief_rgba8", lambda x: calls.append(("rgba8", x)) or torch.ones(3, 4, 4))
    monkeypatch.setattr(E, "raw_body", lambda e, t: calls.append(("raw", e, t)) or torch.zeros(12 * 6, dtype=torch.uint8))
    monkeypatch.setattr(postproc, "to_host", lambda t: calls.append(("to_host",)) or t)
    p = WorldPipeline(native_resolution=30.0)
    p.get_elev, p._get_device, p._relief_on_device = get_elev, get_device, relief

    out = p.get_detail(1, 2, 4, 6, mode="elevation")               # get_elev only: no climate
    assert isinstance(out, np.ndarray) and out.shape == (3, 4, 4)
    assert [c[0] for c in calls] == ["get_elev", "colour", "to_host"]
    assert calls[0][1] == (1, 2, 4, 6) and calls[1][1] is elev and calls[1][2] == "terrain"
    calls.clear()
    p.get_detail(1, 2, 4, 6, mode="temperature")
    assert [c[0] for c in calls] == ["_get_device", "colour", "to_host"]
    assert calls[0][1] == (1, 2, 4, 6, True) and torch.equal(calls[1][1], climate[0]) and calls[1][2] == "RdBu_r"
    for mode in ("relief", "biome", "rgb"):
        calls.clear()
        p.get_detail(1, 2, 4, 6, mode=mode)
        assert [c[0] for c in calls] == ["relief", "rgba8", "to_host"]
        assert calls[0][1:] == ((1, 2, 4, 6), {}) and calls[1][1] is rgb
    calls.clear()
    body, hw, has_temp = p.detail_raw_payload(1, 2, 4, 6)
    assert isinstance(body, bytes) and len(body) == 72 and hw == (3, 4) and has_temp is True
    assert [c[0] for c in calls] == ["_get_device", "raw", "to_host"]
    assert calls[1][1] is elev and torch.equal(calls[1][2], climate[0])
    calls.clear()
    p._host_views = False                                           # TerrainPipeline: the device tensor itself
    assert torch.is_tensor(p.get_detail(1, 2, 4, 6)) and "to_host" not in [c[0] for c in calls]


def test_get_relief_still_returns_host_or_device_arrays(monkeypatch):
    p = WorldPipeline(native_resolution=30.0)
    p._relief_on_device = lambda *win, **kw: torch.ones(2, 3, 3)
    assert isinstance(p.get_relief(0, 0, 2, 3), np.ndarray)
    p._host_views = False
    assert torch.is_tensor(p.get_relief(0, 0, 2, 3))


def test_bench_explorer_help_runs():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_explorer.py"), "--help"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--iters" in out.stdout and "--sizes" in out.stdout
