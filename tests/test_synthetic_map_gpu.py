"""FastNoiseLite Perlin noise and the synthetic conditioning map on the GPU (csrc/tdx_synth.cu through
terrain_diffusion_b200.inference.synthetic_map, the pipelines' `synthetic_map_stats=` and the Minecraft read-out's
`device_noise`).

1. `tdx_fbm_perlin` bit for bit against the numpy restatement (oracle/synthetic_map.py) for the five generators of the
   map at both `frequency_mult` defaults and the five Minecraft configurations, over the case windows (negative, across
   0 and +-2^24, non-square), in guarded NaN-filled buffers.
2. `tdx_synthetic_map` fed the reference's stand-in noise bit for bit against the golden of the reference's own factory
   and pipeline methods, in every mode; on its own noise against the oracle factory.
3. Every argument check of both entry points.
4. A small TerrainPipeline with `synthetic_map_stats=` against the same pipeline given the oracle factory as
   `conditioning_fn`, with imports (their NaN cells carried through the coarse solve) and after change_seed;
   `minecraft_payload(noise_fn=device_noise)` against the oracle
   as `noise_fn`.
"""
from __future__ import annotations

import random
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import synthetic_map as O
from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import TerrainPipeline
from terrain_diffusion_b200.inference import minecraft as M
from terrain_diffusion_b200.inference import synthetic_map as S
from terrain_diffusion_b200.models import EDMUnet2D
from tests import _nonfinite as NF
from tests._igemm_ref import Guarded
from tests._synthetic_inputs import (BIG, CASES, FREQ_ONES, FREQ_SYNTH, IMPORT_CASES, knot_noise, knot_raw,
                                     stand_in_fields, stats_mapping, write_stats)
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG
from tests.test_synthetic_map_cpu import oracle_factory, same_bits

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
G = np.load(Path(__file__).resolve().parent / "golden" / "synthetic_golden.npz")


def run_fbm(configs, i0, j0, h, w) -> np.ndarray:
    out = Guarded((len(configs), h, w), torch.float32, DEV)
    seeds = np.array([S._int32(c[0]) for c in configs], np.int32)
    freq = np.array([c[1] for c in configs], np.float32)
    octv = np.array([c[2] for c in configs], np.int32)
    lac = np.array([c[3] for c in configs], np.float32)
    gain = np.array([c[4] for c in configs], np.float32)
    L.call(L.lib().tdx_fbm_perlin, DEV, len(configs), seeds.ctypes.data, freq.ctypes.data, octv.ctypes.data, lac.ctypes.data,
           gain.ctypes.data, i0, j0, h, w, out.data_ptr())
    torch.cuda.synchronize()
    out.check("fbm_perlin")
    return out.view.cpu().numpy()


FBM_WINDOWS = [CASES[c][3] for c in CASES] + [(-300, -1000, -44, -744), (BIG - 100, BIG - 100, BIG + 156, BIG + 156)]


@pytest.mark.parametrize("fm", [FREQ_SYNTH, FREQ_ONES], ids=["freq_pipeline", "freq_ones"])
@pytest.mark.parametrize("win", FBM_WINDOWS, ids=[f"{w[0]}_{w[1]}_{w[2]}_{w[3]}" for w in FBM_WINDOWS])
def test_fbm_map_generators_match_oracle(fm, win):
    i1, j1, i2, j2 = win
    seeds = O.noise_seeds(abs(hash(win)) % (1 << 40) + 1)
    configs = [(seeds[k], *cfg) for k, cfg in enumerate(O.field_configs(fm))]
    got = run_fbm(configs, j1, i1, j2 - j1, i2 - i1)           # the factory's grid: x = i1 + c, y = j1 + r
    for k, cfg in enumerate(configs):
        want = O.fbm_plane(*cfg, j1, i1, j2 - j1, i2 - i1)
        assert same_bits(got[k], want), (k, cfg)


@pytest.mark.parametrize("win", FBM_WINDOWS, ids=[f"{w[0]}_{w[1]}_{w[2]}_{w[3]}" for w in FBM_WINDOWS])
def test_fbm_minecraft_configs_match_oracle(win):
    i0, j0, i1, j1 = win
    # plus a one-octave, a negative-gain and a many-octave generator; the last octave's coordinate stays below 2^31
    # (0.02 * 1.9^7 * 2^24 ~ 3e7), the range where FastNoiseLite's float-to-int conversion is defined
    configs = list(M.NOISE_CONFIGS) + [(-7, 0.31, 1, 2.5, 0.6), ((1 << 31) - 1, 0.02, 8, 1.9, -0.5)]
    got = run_fbm(configs, i0, j0, i1 - i0, j1 - j0)
    for k, cfg in enumerate(configs):
        assert same_bits(got[k], O.fbm_plane(*cfg, i0, j0, i1 - i0, j1 - j0)), cfg


def test_fbm_public_function():
    got = S.fbm_perlin(4242, 0.05 * 1.5, 4, 2.0, 0.5, -BIG - 3, 17, 40, 70)
    assert got.is_cuda and got.shape == (40, 70)
    assert same_bits(got.cpu().numpy(), O.fbm_plane(4242, 0.05 * 1.5, 4, 2.0, 0.5, -BIG - 3, 17, 40, 70))
    assert same_bits(S.fbm_perlin(1 << 32 | 9, 0.1, 2, 2.0, 0.5, 0, 0, 8, 8).cpu().numpy(),
                     O.fbm_plane(9, 0.1, 2, 2.0, 0.5, 0, 0, 8, 8))
    for bad in [dict(octaves=0), dict(octaves=17), dict(h=0), dict(w=1.5)]:
        args = dict(seed=1, frequency=0.1, octaves=2, lacunarity=2.0, gain=0.5, i0=0, j0=0, h=4, w=4)
        args.update(bad)
        with pytest.raises(ValueError):
            S.fbm_perlin(**args)


# ------------------------------------------------------------------------------------------------ tdx_synthetic_map
def factory(case: str | None = None, seed=None, fm=FREQ_SYNTH) -> S.SyntheticMap:
    if case is not None:
        seed, draw, fm, _ = CASES[case]
        random.seed(draw)
    return S.make_synthetic_map_factory(fm, seed, stats=stats_mapping(), device=DEV)


def run_map(f: S.SyntheticMap, h, w, mode, i0=0, j0=0, noise=None, imports=None, perlin=False) -> np.ndarray:
    """One tdx_synthetic_map launch into a guarded NaN-filled [5, h, w] buffer."""
    out = Guarded((5, h, w), torch.float32, DEV)
    inp = None if noise is None else torch.from_numpy(np.ascontiguousarray(noise, np.float32)).to(DEV)
    tables = None if mode & S.RAW_INPUT else f.tables(DEV)
    imp = S.device_imports(*imports, DEV) if imports is not None else (None, None, None, 0, None)
    L.call(L.lib().tdx_synthetic_map, DEV, None if tables is None else tables.data_ptr(), f.n_knots,
           f._seeds.ctypes.data if perlin else None, f._freq.ctypes.data if perlin else None,
           f._scalars.ctypes.data if mode & S.FINALIZE else None, i0, j0, h, w, None if inp is None else inp.data_ptr(),
           mode, *imp[:4], out.data_ptr())
    torch.cuda.synchronize()
    out.check("synthetic_map")
    return out.view.cpu().numpy()


def stand_in_grid(f: S.SyntheticMap, x0, y0, h, w) -> np.ndarray:
    """fp32 [5, h, w] of the stand-in generators of f's seeds at x = x0 + c, y = y0 + r."""
    xx, yy = np.meshgrid(np.arange(x0, x0 + w, dtype=np.float32), np.arange(y0, y0 + h, dtype=np.float32))
    return np.stack([stand_in_fields(f.seeds[k], 0.05 * f.frequency_mult[k], O.FIELD_OCTAVES[k], 2.0, 0.5, xx, yy)
                     for k in range(5)]).astype(np.float32)


@pytest.mark.parametrize("case", list(CASES))
def test_kernel_with_stand_in_noise_matches_factory_golden(case):
    f = factory(case)
    i1, j1, i2, j2 = CASES[case][3]
    h, w = j2 - j1, i2 - i1
    noise = stand_in_grid(f, i1, j1, h, w)
    raw = run_map(f, h, w, 0, noise=noise).reshape(5, i2 - i1, j2 - j1)
    assert same_bits(raw, G[f"case.{case}.raw"].astype(np.float32))
    full = run_map(f, h, w, S.FINALIZE | S.SQRT0, noise=noise).reshape(5, i2 - i1, j2 - j1)
    assert same_bits(full, G[f"case.{case}.map"])
    # the public form of the injection
    assert same_bits(f.from_noise(torch.from_numpy(noise).to(DEV)).view(5, i2 - i1, j2 - j1).cpu().numpy(),
                     G[f"case.{case}.map"])


@pytest.mark.parametrize("case", list(IMPORT_CASES))
def test_kernel_with_stand_in_noise_matches_import_golden(case):
    (ci0, ci1, cj0, cj1), fcase, imports = IMPORT_CASES[case]
    f = factory(fcase)
    h, w = ci1 - ci0, cj1 - cj0
    noise = stand_in_grid(f, cj0, ci0, h, w)          # sample_raw(cj0, ci0, cj1, ci1): x = cj0 + c, y = ci0 + r
    assert same_bits(run_map(f, h, w, S.FINALIZE | S.SQRT0, noise=noise), G[f"import.{case}.plain"])
    state = ({ch: v for ch, (v, _, _) in imports.items()}, {ch: o for ch, (_, o, _) in imports.items()},
             {ch: d for ch, (_, _, d) in imports.items() if d is not None})
    got = run_map(f, h, w, S.IMPORT | S.SQRT0, ci0, cj0, noise=noise, imports=state)
    assert same_bits(got, G[f"import.{case}"])


def test_kernel_knots_and_finalize_match_golden():
    f = factory(seed=5)
    raw = run_map(f, 8, 16, 0, noise=knot_noise())
    assert same_bits(raw, G["knots.raw"].astype(np.float32))
    fin = run_map(f, 8, 16, S.RAW_INPUT | S.FINALIZE, noise=knot_raw())
    assert same_bits(fin, G["knots.finalize"])
    assert same_bits(f.finalize(knot_raw()).cpu().numpy(), G["knots.finalize"])
    assert same_bits(f.finalize(torch.from_numpy(knot_raw()).to(DEV)[:, 2:5]).cpu().numpy(), G["knots.finalize"][:, 2:5])
    # sqrt alone on a raw input: channel 0 only, zeros of both signs to +0
    both = run_map(f, 8, 16, S.RAW_INPUT | S.SQRT0, noise=knot_raw())
    want = knot_raw().copy()
    want[0] = O.signed_sqrt(want[0])
    assert same_bits(both, want)


@pytest.mark.parametrize("case", list(CASES))
def test_factory_matches_oracle(case):
    f = factory(case)
    o = oracle_factory(case, noise_fn=None)
    assert f.seeds == o.seeds
    win = CASES[case][3]
    raw = f.sample_raw(*win)
    assert raw.is_cuda and same_bits(raw.cpu().numpy(), o.sample_raw(*win).astype(np.float32))
    m = f(*win)
    assert m.is_cuda and m.dtype == torch.float32 and same_bits(m.cpu().numpy(), o(*win))
    i1, j1, i2, j2 = win                                        # the entry point on its own generators
    direct = run_map(f, j2 - j1, i2 - i1, S.FINALIZE | S.SQRT0, j1, i1, perlin=True)
    assert same_bits(direct.reshape(5, i2 - i1, j2 - j1), o(*win))
    assert same_bits(f.finalize(raw).cpu().numpy(), o.finalize(o.sample_raw(*win)))


def test_factory_from_cache_path(tmp_path, monkeypatch):
    write_stats(tmp_path / "s.json")
    f = S.make_synthetic_map_factory(FREQ_ONES, 77, stats=tmp_path / "s.json")
    o = O.Factory(stats_mapping(), FREQ_ONES, 77)
    assert same_bits(f(-5, 3, 27, 35).cpu().numpy(), o(-5, 3, 27, 35))
    monkeypatch.chdir(tmp_path)
    (tmp_path / "data" / "global").mkdir(parents=True)
    write_stats(tmp_path / S.STATS_CACHE_PATH)
    assert same_bits(S.make_synthetic_map_factory(FREQ_ONES, 77)(-5, 3, 27, 35).cpu().numpy(), o(-5, 3, 27, 35))


def test_argument_checks():
    f = factory(seed=3)
    t = f.tables(DEV)
    x = torch.zeros(5 * 64, device=DEV)
    p = x.data_ptr()
    s5, f5, sc = f._seeds.ctypes.data, f._freq.ctypes.data, f._scalars.ctypes.data
    ptrs = np.zeros(5, np.uint64)
    boxes = np.zeros((5, 4), np.int64)
    ptrs[1] = p
    boxes[1] = (0, 0, 0, 4)                                     # an import with no rows
    d5 = np.zeros(5, np.float32)
    one = np.ones(8, np.int32)
    fl = np.full(8, 0.5, np.float32)
    lib = L.lib()
    n = f.n_knots
    cases = [
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, 3, None, None, None, 0, None)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, 16, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, S.RAW_INPUT, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (None, n, s5, f5, sc, 0, 0, 8, 8, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), 1, s5, f5, sc, 0, 0, 8, 8, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), 513, s5, f5, sc, 0, 0, 8, 8, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, None, f5, sc, 0, 0, 8, 8, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, None, sc, 0, 0, 8, 8, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, None, 0, 0, 8, 8, None, 1, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 0, 8, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, -1, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, (1 << 24) + 1, 1, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 1 << 62, 0, 8, 8, None, 3, None, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, 6, None, boxes.ctypes.data, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, 6, ptrs.ctypes.data, None, None, 0, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, 6, ptrs.ctypes.data, boxes.ctypes.data,
                                 None, 1, p)),
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, 6, ptrs.ctypes.data, boxes.ctypes.data,
                                 d5.ctypes.data, 0, p)),                              # the empty import
        (lib.tdx_synthetic_map, (t.data_ptr(), n, s5, f5, sc, 0, 0, 8, 8, None, 3, None, None, d5.ctypes.data, 32, p)),
        (lib.tdx_fbm_perlin, (0, one.ctypes.data, fl.ctypes.data, one.ctypes.data, fl.ctypes.data, fl.ctypes.data, 0, 0,
                              8, 8, p)),
        (lib.tdx_fbm_perlin, (9, one.ctypes.data, fl.ctypes.data, one.ctypes.data, fl.ctypes.data, fl.ctypes.data, 0, 0,
                              8, 8, p)),
        (lib.tdx_fbm_perlin, (1, None, fl.ctypes.data, one.ctypes.data, fl.ctypes.data, fl.ctypes.data, 0, 0, 8, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, None, one.ctypes.data, fl.ctypes.data, fl.ctypes.data, 0, 0, 8, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, None, fl.ctypes.data, fl.ctypes.data, 0, 0, 8, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, one.ctypes.data, None, fl.ctypes.data, 0, 0, 8, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, one.ctypes.data, fl.ctypes.data, None, 0, 0, 8, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, one.ctypes.data, fl.ctypes.data, fl.ctypes.data, 0, 0,
                              8, 8, None)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, np.zeros(1, np.int32).ctypes.data, fl.ctypes.data,
                              fl.ctypes.data, 0, 0, 8, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, np.full(1, 17, np.int32).ctypes.data, fl.ctypes.data,
                              fl.ctypes.data, 0, 0, 8, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, one.ctypes.data, fl.ctypes.data, fl.ctypes.data, 0, 0,
                              0, 8, p)),
        (lib.tdx_fbm_perlin, (1, one.ctypes.data, fl.ctypes.data, one.ctypes.data, fl.ctypes.data, fl.ctypes.data,
                              -(1 << 62), 0, 8, 8, p)),
    ]
    before = x.clone()
    for fn, args in cases:
        with pytest.raises(L.TdxError):
            L.call(fn, DEV, *args)
    torch.cuda.synchronize()
    assert torch.equal(x, before), "a refused call wrote its output"


def test_side_stream_and_repeat():
    f = factory(seed=123)
    first = f(-40, 7, 24, 71)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        again = f(-40, 7, 24, 71)
        noise = S.fbm_perlin(5, 0.3, 3, 2.0, 0.5, 0, 0, 64, 64)
    side.synchronize()
    assert torch.equal(first, again)
    assert same_bits(noise.cpu().numpy(), O.fbm_plane(5, 0.3, 3, 2.0, 0.5, 0, 0, 64, 64))


# ------------------------------------------------------------------------------------------------------ pipelines
def _models():
    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.cuda()
    return build(COARSE_CFG), build(BASE_CFG), build(ounet.DECODER_CFG)


def _pipeline(models, **kw):
    g = torch.Generator().manual_seed(3)
    return TerrainPipeline(*models, seed=kw.pop("seed", 20261017), coarse_means=(torch.randn(6, generator=g) * 0.1).tolist(),
                           coarse_stds=(torch.rand(6, generator=g) + 0.5).tolist(), cond_snr=[0.3, 0.5, 1.0, 2.0, 4.0],
                           histogram_raw=torch.randn(5, generator=g), latents_means=torch.zeros(7),
                           latents_stds=torch.ones(7), decoder_tile_size=128, decoder_tile_stride=96,
                           residual_mean=0.1, residual_std=1.2, native_resolution=30.0, **kw)


def test_pipeline_synthesis_matches_oracle_conditioning_and_keeps_nodata():
    """Default mode, after change_seed, and with imports whose NaN (nodata) cells the coarse solve carries through,
    as the reference's does."""
    models = _models()
    stats = stats_mapping()
    dev_pipe = _pipeline(models, synthetic_map_stats=stats)
    imports: dict = {}
    ref_pipe = None

    def cond_fn(i1, i2, j1, j2):                       # the reference's _conditioning_model_input through the oracle
        f = O.Factory(stats, FREQ_SYNTH, ref_pipe.seed)
        if imports:
            return torch.from_numpy(O.import_conditioning(f, imports, i1, i2, j1, j2))
        return torch.from_numpy(f(j1, i1, j2, i2))

    ref_pipe = _pipeline(models, conditioning_fn=cond_fn)
    win = (slice(None), slice(-40, 70), slice(-100, 10))

    def check(what, nodata=False):
        a, b = dev_pipe.coarse[win], ref_pipe.coarse[win]
        assert a.is_cuda, what
        # the reference's coarse solve carries an imported raster's NaN (nodata) cells through unfiltered (the clip of
        # every U-Net block keeps NaN, as torch.clip does); without them the canvas is finite
        assert bool(torch.isnan(a).any()) == nodata and not bool(torch.isinf(a).any()), what
        NF.assert_same_bits(a, b, what)

    for i, j in [(0, 0), (-1, 2), (3, -4)]:
        smap = dev_pipe._conditioning_model_input(48 * i, 48 * i + 64, 48 * j, 48 * j + 64)
        assert smap.is_cuda and same_bits(smap.cpu().numpy(), cond_fn(48 * i, 48 * i + 64, 48 * j, 48 * j + 64).numpy())
    check("default mode")
    for p in (dev_pipe, ref_pipe):
        assert p.change_seed((1 << 64) - 5)
    assert dev_pipe._synthetic.seeds == O.noise_seeds((1 << 64) - 5)
    check("after change_seed")
    values = np.random.default_rng(1).uniform(-2000, 3000, (70, 50)).astype(np.float32)
    values[::7, ::5] = np.nan
    values[3::11, 1::9] = -0.0
    temp = np.random.default_rng(2).uniform(-5, 25, (30, 30)).astype(np.float32)
    dev_pipe.set_custom_conditioning_import(0, values, -60, -80)
    dev_pipe.set_custom_conditioning_import(1, temp, 20, -30, default_value=14.0)
    imports.update({0: (values, (-60, -80), None), 1: (temp, (20, -30), 14.0)})
    ref_pipe.rebuild()
    for i, j in [(0, 0), (-1, -2)]:
        smap = dev_pipe._conditioning_model_input(48 * i, 48 * i + 64, 48 * j, 48 * j + 64)
        assert same_bits(smap.cpu().numpy(), cond_fn(48 * i, 48 * i + 64, 48 * j, 48 * j + 64).numpy())
    check("with imports", nodata=True)


def test_pipeline_frequency_mult_and_default_get():
    stats = stats_mapping()
    models = _models()
    p = _pipeline(models, synthetic_map_stats=stats, frequency_mult=[1, 1, 2, 1, 1], seed=99)
    smap = p._conditioning_model_input(-64, 0, 0, 64)
    assert same_bits(smap.cpu().numpy(), O.Factory(stats, [1, 1, 2, 1, 1], 99)(0, -64, 64, 0))
    out = p.get(-64, -32, 64, 96)
    assert torch.isfinite(out["elev"]).all() and torch.isfinite(out["climate"]).all()
    # the Minecraft read-out with the device noise provider is byte for byte the one with the oracle's noise
    for scale in (1, 2):
        body, hw = p.minecraft_payload(-20, 10, 12, 42, scale=scale, noise_fn=M.device_noise)
        want, hw2 = p.minecraft_payload(-20, 10, 12, 42, scale=scale,
                                        noise_fn=lambda cfg, i0, j0, h, w: O.fbm_plane(*cfg, i0, j0, h, w))
        assert hw == hw2 == (32, 32) and body == want


def test_minecraft_device_noise_matches_oracle():
    from tests._minecraft_inputs import BiomeWorld
    world = BiomeWorld(seed=4)

    def get_device(i1, j1, i2, j2, with_climate=True):
        out = world.get(i1, j1, i2, j2, with_climate)
        return {k: (None if v is None else v.to(DEV)) for k, v in out.items()}

    def oracle_noise(cfg, i0, j0, h, w):
        return O.fbm_plane(*cfg, i0, j0, h, w)

    calls = []

    def counting(cfg, i0, j0, h, w):
        calls.append(cfg)
        return M.device_noise(cfg, i0, j0, h, w)

    for win, scale, noise in [((-20, 10, 44, 90), 1, 1.0), ((-37, -5, -21, 11), 4, 1.0), ((3, -77, 40, 60), 2, 0.0),
                              ((-130, 7, 70, 80), 8, 1.0), ((-BIG, BIG - 40, -BIG + 64, BIG + 24), 2, 1.0)]:
        want, hw = M.request(get_device, 90.0, *win, scale, noise, oracle_noise, payload=True)
        got, hw2 = M.request(get_device, 90.0, *win, scale, noise, M.device_noise, payload=True)
        assert hw == hw2 and torch.equal(got, want), (win, scale, noise)
        counted, _ = M.request(get_device, 90.0, *win, scale, noise, counting, payload=True)
        assert torch.equal(counted, want) and len(calls) == (5 if scale > 1 and noise > 0 else 3)
        calls.clear()
        planes = M.noise_planes(M.device_noise, win[0], win[1], 16, 24, (3, 4), DEV).cpu().numpy()
        assert not planes[:3].any()
        for k in (3, 4):
            assert same_bits(planes[k], O.fbm_plane(*M.NOISE_CONFIGS[k], win[0], win[1], 16, 24))
