"""The explorer's detail view on the GPU (csrc/tdx_explorer.cu through terrain_diffusion_b200.inference.explorer and
`WorldPipeline.get_detail` / `detail_raw_payload`).

1. Every golden of the reference's own handlers (tests/golden/explorer_golden.npz) bit for bit through the C entry
   points: the range into a guarded buffer whose slack starts as garbage, the uint8 images and the raw bodies into
   guarded buffers written twice, over 0x00 and over 0xFF, which must agree (so every byte is written).
2. The public functions against the oracle (oracle/explorer.py) at 512², 1024² and 2048², exactly; CUDA and numpy
   inputs, repeated calls, a side stream and a second device give identical results.
3. A small TerrainPipeline: the elevation image from `get_elev` equals the one from the full `get()`, and every mode
   and the raw body equal the oracle on `get()`'s output; a PIL PNG round trip decodes to the same pixels.
"""
from __future__ import annotations

import io
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import explorer as O
from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import TerrainPipeline, get_relief_map
from terrain_diffusion_b200.inference import explorer as E
from terrain_diffusion_b200.inference.pipeline import WorldPipeline
from terrain_diffusion_b200.models import EDMUnet2D
from tests._explorer_inputs import HANDLER_CASES, NATIVE_RESOLUTION, PLANE_CASES, plane_case, world_planes
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
G = np.load(Path(__file__).resolve().parent / "golden" / "explorer_golden.npz")
PAD = 64


def guarded_bytes(nbytes: int, launch) -> np.ndarray:
    """launch(ptr) into an nbytes buffer with PAD sentinel bytes on each side, twice (over 0x00 and 0xFF); returns the
    bytes after checking the sentinels and that both runs agree."""
    runs = []
    for fill in (0x00, 0xFF):
        raw = torch.full((nbytes + 2 * PAD,), 0x5A, dtype=torch.uint8, device=DEV)
        body = raw[PAD:PAD + nbytes]
        body.fill_(fill)
        launch(body.data_ptr())
        torch.cuda.synchronize()
        assert bool((raw[:PAD] == 0x5A).all()) and bool((raw[PAD + nbytes:] == 0x5A).all()), "written outside the buffer"
        runs.append(body.cpu().numpy())
    assert np.array_equal(runs[0], runs[1]), "some bytes were not written"
    return runs[0]


def run_colour(plane: np.ndarray, cmap: str) -> np.ndarray:
    x = torch.from_numpy(np.ascontiguousarray(plane, np.float32)).to(DEV)
    n = x.numel()
    rng_raw = torch.full((16,), 0x7A5A5A5A, dtype=torch.int32, device=DEV)   # garbage before the call zeroes it
    rng = rng_raw[4:6]
    L.call(L.lib().tdx_detail_range, DEV, x.data_ptr(), n, rng.data_ptr())
    torch.cuda.synchronize()
    assert bool((rng_raw[:4] == 0x7A5A5A5A).all()) and bool((rng_raw[6:] == 0x7A5A5A5A).all())
    lut = E._lut_on(cmap, DEV)
    img = guarded_bytes(4 * n, lambda p: L.call(L.lib().tdx_detail_colour, DEV, x.data_ptr(), n, rng.data_ptr(),
                                                 lut.data_ptr(), p))
    return img.reshape(*plane.shape, 4)


def run_rgba8(rgb: np.ndarray) -> np.ndarray:
    x = torch.from_numpy(np.ascontiguousarray(rgb, np.float32)).to(DEV)
    n = rgb.shape[0] * rgb.shape[1]
    return guarded_bytes(4 * n, lambda p: L.call(L.lib().tdx_detail_rgba8, DEV, x.data_ptr(), n, p)).reshape(
        *rgb.shape[:2], 4)


def run_raw(elev: np.ndarray, temp) -> bytes:
    e = torch.from_numpy(np.ascontiguousarray(elev, np.float32)).to(DEV)
    t = None if temp is None else torch.from_numpy(np.ascontiguousarray(temp, np.float32)).to(DEV)
    n = e.numel()
    return guarded_bytes(n * (2 if t is None else 6), lambda p: L.call(
        L.lib().tdx_detail_raw, DEV, e.data_ptr(), None if t is None else t.data_ptr(), n, p)).tobytes()


def case_window(args):
    return O.detail_window(args.get("ci", 0), args.get("cj", 0), args.get("detail_size", 1024), args.get("pan_i", 0),
                           args.get("pan_j", 0))


@pytest.mark.parametrize("name", list(HANDLER_CASES))
def test_kernels_match_handler_golden(name):
    kind, endpoint, args = HANDLER_CASES[name]
    elev, climate = world_planes(kind, *case_window(args))
    if endpoint == "raw":
        body = run_raw(elev, climate[0])
        assert body == G[f"{name}.body"].tobytes()
        assert run_raw(elev, None) == body[:2 * elev.size]
        return
    mode = args.get("mode", "relief")
    if mode == "elevation":
        got = run_colour(elev, "terrain")
    elif mode == "temperature":
        got = run_colour(climate[0], "RdBu_r")
    else:
        got = run_rgba8(G[f"{name}.relief_rgb"])
    assert np.array_equal(got, G[f"{name}.image"]), f"{name}: {int((got != G[f'{name}.image']).any(-1).sum())} px differ"


@pytest.mark.parametrize("name", list(PLANE_CASES))
def test_kernels_match_plane_golden(name):
    plane, cmap = plane_case(name)
    got = run_colour(plane, cmap)
    assert np.array_equal(got, G[f"plane.{name}.image"])


def test_argument_checks():
    x = torch.zeros(8, device=DEV)
    p = x.data_ptr()
    lib = L.lib()
    for fn, args in [(lib.tdx_detail_range, (p, 0, p)), (lib.tdx_detail_range, (None, 4, p)),
                     (lib.tdx_detail_colour, (p, 4, p, p, p + 1)), (lib.tdx_detail_colour, (p, 4, None, p, p)),
                     (lib.tdx_detail_rgba8, (p, 2, p + 2)), (lib.tdx_detail_rgba8, (p, 0, p)),
                     (lib.tdx_detail_raw, (p, None, 4, p + 1)), (lib.tdx_detail_raw, (None, p, 4, p))]:
        with pytest.raises(L.TdxError):
            L.call(fn, DEV, *args)


# ------------------------------------------------------------------------------------------- public functions at size
SIZES = [512, 1024, 2048]


class PlaneWorld(WorldPipeline):
    """A WorldPipeline whose read-out returns the analytic planes of tests/_explorer_inputs.py on the device."""

    def __init__(self):
        super().__init__(native_resolution=NATIVE_RESOLUTION)
        self.reads = []

    def _planes(self, i1, j1, i2, j2):
        e, c = world_planes("mixed", i1, j1, i2, j2)
        return torch.from_numpy(e).to(DEV), torch.from_numpy(c).to(DEV)

    def get_elev(self, i1, j1, i2, j2, *a, **k):
        self.reads.append("elev")
        return self._planes(i1, j1, i2, j2)[0]

    def _get_device(self, i1, j1, i2, j2, with_climate=True):
        self.reads.append("climate")
        e, c = self._planes(i1, j1, i2, j2)
        return {"elev": e, "climate": c if with_climate else None}


@pytest.mark.parametrize("n", SIZES)
def test_public_methods_match_oracle(n):
    win = (-(n // 3), 77, n - n // 3, 77 + n)
    elev, climate = world_planes("mixed", *win)
    world = PlaneWorld()
    got = world.get_detail(*win, mode="elevation")
    assert isinstance(got, np.ndarray) and got.shape == (n, n, 4) and world.reads == ["elev"]
    assert np.array_equal(got, O.colour_plane(elev, "terrain"))
    assert np.array_equal(world.get_detail(*win, mode="temperature"), O.colour_plane(climate[0], "RdBu_r"))
    relief = world.get_detail(*win)
    rgb = get_relief_map(elev, None, None, None, resolution=NATIVE_RESOLUTION)
    assert np.array_equal(relief, O.relief_rgba(rgb))
    assert relief[..., 3].min() == 255
    body, hw, has_temp = world.detail_raw_payload(*win)
    assert hw == (n, n) and has_temp and body == O.detail_raw_body(elev, climate[0])
    for cmap, plane in (("terrain", elev), ("RdBu_r", climate[0])):
        d = torch.from_numpy(plane).to(DEV)
        a = E.colour_plane(d, cmap)
        assert a.is_cuda and a.dtype == torch.uint8 and tuple(a.shape) == (n, n, 4)
        assert np.array_equal(a.cpu().numpy(), O.colour_plane(plane, cmap))


def test_input_kinds_streams_and_devices():
    elev, climate = world_planes("nan_temp", 0, 0, 300, 257)
    temp = climate[0]
    host = E.colour_plane(temp, "RdBu_r")
    assert isinstance(host, np.ndarray) and np.array_equal(host, O.colour_plane(temp, "RdBu_r"))
    assert np.array_equal(E.colour_plane(torch.from_numpy(temp), "RdBu_r"), host)        # CPU tensor in, numpy out
    d = torch.from_numpy(temp).to(DEV)
    first = E.colour_plane(d, "RdBu_r")
    for _ in range(3):
        assert torch.equal(E.colour_plane(d, "RdBu_r"), first)
    assert np.array_equal(first.cpu().numpy(), host)
    assert torch.equal(E.colour_plane(d.t().contiguous().t(), "RdBu_r"), first)           # strided input
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        img = E.colour_plane(d, "RdBu_r")
        body = E.raw_body(torch.from_numpy(elev).to(DEV), d)
    side.synchronize()
    assert torch.equal(img, first)
    assert body.cpu().numpy().tobytes() == O.detail_raw_body(elev, temp)
    if torch.cuda.device_count() > 1:
        d1 = d.to("cuda:1")
        img1 = E.colour_plane(d1, "RdBu_r")
        assert img1.device == d1.device and torch.equal(img1.cpu(), first.cpu())
        rgb1 = torch.rand(5, 6, 3, device="cuda:1")
        assert torch.equal(E.relief_rgba8(rgb1).cpu(), torch.from_numpy(O.relief_rgba(rgb1.cpu().numpy())))


# ------------------------------------------------------------------------------------------------------ pipeline
@pytest.fixture(scope="module")
def pipe():
    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.cuda()

    def cond_fn(i1, i2, j1, j2):
        gg = torch.Generator().manual_seed(i1 * 7919 + j1 + 12345)
        return torch.randn(5, i2 - i1, j2 - j1, generator=gg)

    g = torch.Generator().manual_seed(3)
    return TerrainPipeline(build(COARSE_CFG), build(BASE_CFG), build(ounet.DECODER_CFG), seed=7, conditioning_fn=cond_fn,
                           coarse_means=(torch.randn(6, generator=g) * 0.1).tolist(),
                           coarse_stds=(torch.rand(6, generator=g) + 0.5).tolist(), cond_snr=[0.3, 0.5, 1.0, 2.0, 4.0],
                           histogram_raw=torch.randn(5, generator=g), latents_means=torch.zeros(7),
                           latents_stds=torch.ones(7), decoder_tile_size=128, decoder_tile_stride=96,
                           residual_mean=0.1, residual_std=1.2, native_resolution=30.0)


@pytest.mark.parametrize("win", [(-20, 10, 44, 90), (-150, -37, -100, 9)])
def test_terrain_pipeline_detail_view(pipe, win):
    region = pipe.get(*win)
    elev, temp = region["elev"].cpu().numpy(), region["climate"][0].cpu().numpy()
    img = pipe.get_detail(*win, mode="elevation")
    assert img.is_cuda and img.dtype == torch.uint8 and tuple(img.shape) == elev.shape + (4,)
    assert torch.equal(img, E.colour_plane(region["elev"], "terrain"))     # get_elev alone == the full get()
    assert np.array_equal(img.cpu().numpy(), O.colour_plane(elev, "terrain"))
    assert np.array_equal(pipe.get_detail(*win, mode="temperature").cpu().numpy(), O.colour_plane(temp, "RdBu_r"))
    relief = pipe.get_detail(*win, mode="relief")
    assert torch.equal(relief, pipe.get_detail(*win, mode="anything else"))
    assert torch.equal(relief, E.relief_rgba8(pipe.get_relief(*win)))
    body, hw, has_temp = pipe.detail_raw_payload(*win)
    assert hw == elev.shape and has_temp and body == O.detail_raw_body(elev, temp)
    pipe._host_views = True                                    # WorldPipeline: numpy through one pinned copy
    try:
        host = pipe.get_detail(*win, mode="temperature")
    finally:
        pipe._host_views = False
    assert isinstance(host, np.ndarray) and np.array_equal(host, O.colour_plane(temp, "RdBu_r"))


def test_png_round_trip(pipe):
    from PIL import Image
    for mode in ("elevation", "temperature", "relief"):
        img = pipe.get_detail(-20, 10, 44, 90, mode=mode).cpu().numpy()
        buf = io.BytesIO()
        Image.fromarray(img, "RGBA").save(buf, format="png")
        buf.seek(0)
        assert np.array_equal(np.asarray(Image.open(buf).convert("RGBA")), img)
    nan_img = G["nan_relief.image"]                           # transparent pixels survive the encoder too
    buf = io.BytesIO()
    Image.fromarray(nan_img, "RGBA").save(buf, format="png")
    buf.seek(0)
    assert np.array_equal(np.asarray(Image.open(buf)), nan_img)
