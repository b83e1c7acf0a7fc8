"""The explorer's coarse map and the random sampler's land search on the GPU (csrc/tdx_coarse_view.cu through
terrain_diffusion_b200.inference.coarse_view and the `WorldPipeline` methods).

1. Every golden of the reference's own functions (tests/golden/coarse_view_golden.npz) through the C entry points: the
   planes bit for bit against the oracle except channel 4's log1p display plane, which is within 2 ulp of numpy's fp32
   log1p (neither is correctly rounded); the image bit for bit against the oracle fed the device's display plane, and
   against the golden itself; range buffers whose slack starts as garbage; images and tile lists in
   guarded buffers written twice, over 0x00 and over 0xFF, which must agree.
2. The land search at detail sizes 256 (empty window), 768, 1024 and 8192 and min_land_frac 0, 0.5 and 1 over a
   600 x 600 coarse window, against the oracle.
3. The public methods on a world of analytic sums and on a small TerrainPipeline against `coarse[...]` + the oracle;
   the sampler drop-ins under random.seed(k) against the reference's picks.
"""
from __future__ import annotations

import random
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import coarse_view as O
from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import TerrainPipeline
from terrain_diffusion_b200.inference import coarse_view as CV
from terrain_diffusion_b200.inference.pipeline import WorldPipeline
from terrain_diffusion_b200.models import EDMUnet2D
from tests._coarse_view_inputs import (CLIMATE_CELLS, DATA_CASES, LAND_CASES, LAND_WINDOW, PNG_CASES, SAMPLE_CASES,
                                       seeded_lut, world_sums)
from tests.test_coarse_view_cpu import WINDOW, png_args
from tests.test_explorer_gpu import guarded_bytes
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
G = np.load(Path(__file__).resolve().parent / "golden" / "coarse_view_golden.npz")
GARBAGE = 0x7A5A5A5A


def lut_dev():
    return torch.from_numpy(seeded_lut().astype(np.float32)).to(DEV)


def run_readout(sums: np.ndarray, eps: bool):
    """(planes fp32 [7, h, w], range keys int32 [14]) through tdx_coarse_readout, range in a garbage-filled buffer."""
    s = torch.from_numpy(np.ascontiguousarray(sums, np.float32)).to(DEV)
    n = s.shape[1] * s.shape[2]
    planes = torch.full((7, *s.shape[1:]), float("nan"), device=DEV)
    rng_raw = torch.full((20,), GARBAGE, dtype=torch.int32, device=DEV)
    rng = rng_raw[3:17]
    L.call(L.lib().tdx_coarse_readout, DEV, s.data_ptr(), n, int(eps), planes.data_ptr(), rng.data_ptr())
    torch.cuda.synchronize()
    assert bool((rng_raw[:3] == GARBAGE).all()) and bool((rng_raw[17:] == GARBAGE).all())
    # the range-only launch gives the same keys
    rng2 = torch.full((14,), GARBAGE, dtype=torch.int32, device=DEV)
    L.call(L.lib().tdx_coarse_readout, DEV, s.data_ptr(), n, int(eps), None, rng2.data_ptr())
    assert torch.equal(rng2, rng)
    return planes, rng


def run_image(planes: torch.Tensor, rng: torch.Tensor, channel: int, filters) -> np.ndarray:
    bounds, active = CV.filter_bounds(filters)
    lut = lut_dev()
    h, w = planes.shape[1:]
    b = np.ascontiguousarray(bounds, np.float32)
    img = guarded_bytes(4 * h * w, lambda p: L.call(L.lib().tdx_coarse_image, DEV, planes.data_ptr(), h * w, channel,
                                                    rng.data_ptr(), lut.data_ptr(), b.ctypes.data, active, p))
    return img.reshape(h, w, 4)


def ulp_distance(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    def ordered(x):
        i = x.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


def check_planes(planes: torch.Tensor, sums: np.ndarray, eps: bool) -> np.ndarray:
    """The device planes against the oracle: channels 0..5 bit for bit, the display plane within 1 ulp."""
    got = planes.cpu().numpy()
    want = O.coarse_planes(sums, eps)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got[:6]), nan)
    assert np.array_equal(got[:6][~nan].view(np.uint32), want[~nan].view(np.uint32))     # signed zeros included
    shown = O.display(want, 4)
    assert np.array_equal(np.isnan(got[6]), np.isnan(shown))
    fin = ~np.isnan(shown)
    # numpy's fp32 log1p is not correctly rounded: 11783 of the 360000 cells of the 600^2 sampler window are 2 ulp off
    # the correctly rounded value on an AVX-512 host, so the two single-precision log1p's can differ by 2 ulp
    assert int(ulp_distance(got[6][fin], shown[fin]).max(initial=0)) <= 2
    return got


@pytest.mark.parametrize("name", list(PNG_CASES))
def test_kernels_match_png_golden(name):
    kind, args = PNG_CASES[name]
    win, channel, filters = png_args(args)
    sums = world_sums(kind, *win)
    planes, rng = run_readout(sums, True)
    got_planes = check_planes(planes, sums, True)
    img = run_image(planes, rng, channel, filters)
    want, vmin, vmax = O.coarse_image(O.coarse_planes(sums), channel, seeded_lut(), filters,
                                      shown=got_planes[6] if channel == 4 else None)
    assert np.array_equal(img, want)
    assert CV.display_range(rng, channel) == (vmin, vmax) or all(np.isnan([vmin, vmax]))
    assert [str(round(v, 3)) for v in CV.display_range(rng, channel)] == G[f"png.{name}.headers"].tolist()
    assert np.array_equal(img, G[f"png.{name}.image"])


@pytest.mark.parametrize("name", list(DATA_CASES))
def test_kernels_match_data_and_stats_golden(name):
    kind, win = DATA_CASES[name]
    sums = world_sums(kind, *(win[k] for k in WINDOW))
    planes, rng = run_readout(sums, True)
    check_planes(planes, sums, True)
    n = planes[:6].numel()
    out = torch.from_numpy(guarded_bytes(4 * n, lambda p: L.call(L.lib().tdx_coarse_round, DEV, planes.data_ptr(), n,
                                                                    p)).view(np.float32).reshape(6, *planes.shape[1:]))
    assert np.array_equal(out.numpy().astype(np.float64), G[f"data.{name}"], equal_nan=True)
    ranges = CV.range_values(rng)
    got = np.array([[round(ranges[c][0], 3), round(ranges[c][1], 3)] for c in range(6)])
    assert np.array_equal(got, G[f"stats.{name}"], equal_nan=True)


def run_land(elev_m: torch.Tensor, half: int, frac: float) -> list:
    """Window centres (i, j) through tdx_coarse_land.  The list goes into a buffer with sentinels on both sides, twice
    (over 0 and over -1): the count and the indices it covers must agree, and match the mask's row-major compaction."""
    h, w = elev_m.shape
    ho, wo = h - 2 * half, w - 2 * half
    n = max(ho, 0) * max(wo, 0)
    rows = torch.empty((h, max(wo, 1)), dtype=torch.int32, device=DEV)
    mask = torch.empty(max(n, 1), dtype=torch.uint8, device=DEV)
    runs = []
    for fill in (0, -1):
        raw = torch.full((1 + n + 32,), GARBAGE, dtype=torch.int32, device=DEV)
        lst = raw[16:17 + n]
        lst.fill_(fill)
        L.call(L.lib().tdx_coarse_land, DEV, elev_m.data_ptr(), h, w, half, frac, rows.data_ptr(), mask.data_ptr(),
               lst.data_ptr())
        host = raw.cpu().numpy()
        assert (host[:16] == GARBAGE).all() and (host[17 + n:] == GARBAGE).all(), "written outside the list"
        count = int(host[16])
        assert 0 <= count <= n
        runs.append(host[16:17 + count])
    assert np.array_equal(runs[0], runs[1])
    idx = runs[0][1:].astype(np.int64)
    if n:
        assert np.array_equal(np.nonzero(mask.cpu().numpy()[:n])[0], idx)
    return [(half + int(k) // max(wo, 1), half + int(k) % max(wo, 1)) for k in idx]


@pytest.mark.parametrize("cw,detail,frac", LAND_CASES)
def test_land_kernel_matches_reference_golden(cw, detail, frac):
    planes, _ = run_readout(world_sums("mixed", -cw, cw, -cw, cw), False)
    tiles = [(i - cw, j - cw) for i, j in run_land(planes[0].contiguous(), (detail // 256) // 2, frac)]
    assert np.array_equal(np.array(tiles, np.int64).reshape(-1, 2), G[f"land.{cw}.{detail}.{frac}"])


@pytest.mark.parametrize("detail", [256, 768, 1024, 8192])
@pytest.mark.parametrize("frac", [0.0, 0.5, 1.0])
def test_land_search_at_the_sampler_defaults(detail, frac):
    cw = 300
    sums = world_sums("mixed", -cw, cw, -cw, cw)
    planes, _ = run_readout(sums, False)
    check_planes(planes, sums, False)
    tiles = [(i - cw, j - cw) for i, j in run_land(planes[0].contiguous(), (detail // 256) // 2, frac)]
    want = O.land_tiles(sums, -cw, -cw, detail, frac)
    assert tiles == want
    if detail > 256 and frac < 1.0:
        assert want


def test_argument_checks():
    x = torch.zeros(64, device=DEV)
    p = x.data_ptr()
    b = np.zeros(12, np.float32)
    lib = L.lib()
    for fn, args in [(lib.tdx_coarse_readout, (p, 0, 1, p, p)), (lib.tdx_coarse_readout, (None, 4, 1, p, p)),
                     (lib.tdx_coarse_readout, (p, 4, 1, p, None)),
                     (lib.tdx_coarse_image, (p, 4, 6, p, p, b.ctypes.data, 0, p)),
                     (lib.tdx_coarse_image, (p, 4, -1, p, p, b.ctypes.data, 0, p)),
                     (lib.tdx_coarse_image, (p, 4, 0, p, p, b.ctypes.data, 1 << 2, p)),      # a channel-1 filter
                     (lib.tdx_coarse_image, (p, 4, 0, p, p, b.ctypes.data, 1 << 12, p)),
                     (lib.tdx_coarse_image, (p, 4, 0, p, p, None, 1, p)),
                     (lib.tdx_coarse_image, (p, 4, 0, p, p, None, 0, p + 1)),
                     (lib.tdx_coarse_round, (p, 0, p)), (lib.tdx_coarse_round, (None, 4, p)),
                     (lib.tdx_coarse_land, (p, 0, 4, 1, 0.5, p, p, p)), (lib.tdx_coarse_land, (p, 4, 4, -1, 0.5, p, p, p)),
                     (lib.tdx_coarse_land, (p, 8, 8, 1, 0.5, None, p, p)), (lib.tdx_coarse_land, (None, 8, 8, 1, 0.5, p, p, p))]:
        with pytest.raises(L.TdxError):
            L.call(fn, DEV, *args)


# ------------------------------------------------------------------------------------------------- public methods
class SumsWorld(WorldPipeline):
    """A WorldPipeline whose coarse canvas returns the analytic sums of tests/_coarse_view_inputs.py on the device."""

    def __init__(self, kind="mixed"):
        super().__init__(native_resolution=30.0)
        self.kind, self.reads = kind, []

    def _coarse_sums(self, ci0, ci1, cj0, cj1):
        self.reads.append((ci0, ci1, cj0, cj1))
        return torch.from_numpy(world_sums(self.kind, ci0, ci1, cj0, cj1)).to(DEV)


@pytest.mark.parametrize("n", [100, 600])
def test_public_methods_match_oracle(n):
    win = (-(n // 3), n - n // 3, 17, 17 + n)
    world = SumsWorld("nan")
    sums = world_sums("nan", *win)
    planes = O.coarse_planes(sums)
    got = world.get_coarse(*win)
    assert isinstance(got, torch.Tensor) and not got.is_cuda and got.dtype == torch.float32
    assert np.array_equal(got.numpy(), planes, equal_nan=True)
    assert np.array_equal(world.get_coarse(*win, eps=False).numpy(), O.coarse_planes(sums, eps=False), equal_nan=True)
    shown = CV.readout(world._coarse_sums(*win))[0][6].cpu().numpy()
    for channel, filters in [(0, None), (2, {0: (0.0, None), 1: (5.0, 6.0)}), (4, {3: (200.0, 400.0)}),
                             (5, {2: (None, 20.0), 4: (100.0, None), 5: (30.0, 70.0)})]:
        img, vmin, vmax = world.coarse_image(*win, channel=channel, filters=filters, lut=seeded_lut())
        want = O.coarse_image(planes, channel, seeded_lut(), filters, shown=shown if channel == 4 else None)
        assert isinstance(img, np.ndarray) and img.shape == (n, n, 4)
        assert np.array_equal(img, want[0]) and (vmin, vmax) == want[1:]
    data = world.coarse_data(*win)
    assert [data[k] for k in WINDOW] == list(win) and list(data["channels"]) == O.CHANNEL_NAMES
    rounded = O.coarse_data(planes)
    for i, name in enumerate(O.CHANNEL_NAMES):
        assert np.array_equal(np.array(data["channels"][name]), rounded[i].astype(np.float64), equal_nan=True)
    stats = world.coarse_stats(*win)
    want_stats = O.coarse_stats(planes)
    assert list(stats) == list(range(6))
    for c in range(6):
        assert stats[c]["name"] == want_stats[c]["name"]
        assert np.array_equal([stats[c]["min"], stats[c]["max"]], [want_stats[c]["min"], want_stats[c]["max"]],
                              equal_nan=True)


@pytest.mark.parametrize("seed,detail,frac,n", SAMPLE_CASES)
def test_sampler_drop_ins_match_reference(seed, detail, frac, n):
    world = SumsWorld("mixed")
    random.seed(seed)
    pick = CV.sample_land_tiles(world, LAND_WINDOW, detail, frac, n)
    assert np.array_equal(np.array(pick, np.int64).reshape(-1, 2), G[f"sample.{seed}"])
    assert world.reads == [(-LAND_WINDOW, LAND_WINDOW, -LAND_WINDOW, LAND_WINDOW)]


@pytest.mark.parametrize("ci,cj", CLIMATE_CELLS)
def test_climate_info_matches_reference(ci, cj):
    info = CV.get_coarse_climate_info(SumsWorld("nan"), ci, cj)
    assert np.array_equal(list(info.values()), G[f"climate.{ci}.{cj}"], equal_nan=True)


def test_side_stream_and_repeat():
    world = SumsWorld("nan")
    win = (-30, 40, -5, 61)
    first = world.coarse_image(*win, channel=4, filters={0: (0.0, None)}, lut=seeded_lut())
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        again = world.coarse_image(*win, channel=4, filters={0: (0.0, None)}, lut=seeded_lut())
        tiles = world.land_tiles(30, 1024, 0.5)
    side.synchronize()
    assert np.array_equal(first[0], again[0]) and first[1:] == again[1:]
    assert tiles == O.land_tiles(world_sums("nan", -30, 30, -30, 30), -30, -30, 1024, 0.5)


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


def test_terrain_pipeline_coarse_view(pipe):
    win = (-40, 37, -25, 60)
    sums = pipe.coarse[:, win[0]:win[1], win[2]:win[3]].cpu().numpy()
    planes = O.coarse_planes(sums)
    got = pipe.get_coarse(*win)
    assert got.is_cuda and np.array_equal(got.cpu().numpy(), planes, equal_nan=True)
    shown = CV.readout(pipe._coarse_sums(*win))[0][6].cpu().numpy()
    img, vmin, vmax = pipe.coarse_image(*win, channel=4, filters={0: (0.0, None), 2: (None, 25.0)}, lut=seeded_lut())
    want = O.coarse_image(planes, 4, seeded_lut(), {0: (0.0, None), 2: (None, 25.0)}, shown=shown)
    assert img.is_cuda and np.array_equal(img.cpu().numpy(), want[0]) and (vmin, vmax) == want[1:]
    stats = pipe.coarse_stats(*win)
    assert stats == O.coarse_stats(planes)
    cw = 30
    tiles = pipe.land_tiles(cw, 1024, 0.5)
    assert tiles == O.land_tiles(pipe.coarse[:, -cw:cw, -cw:cw].cpu().numpy(), -cw, -cw, 1024, 0.5)
    assert pipe.land_tiles(cw, 256, 0.0) == []
    info = CV.get_coarse_climate_info(pipe, 3, -4)
    assert info == O.climate_info(pipe.coarse[:, 3:4, -4:-3].cpu().numpy())
