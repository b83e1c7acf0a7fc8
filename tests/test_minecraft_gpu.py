"""Minecraft API read-out on the GPU (csrc/tdx_biome.cu `tdx_minecraft_readout`, `WorldPipeline.get_minecraft` /
`minecraft_payload`).

1. The C entry point, every fp32 output in a guarded NaN-filled buffer and the int16 outputs written twice over 0x00-
   and 0xFF-filled buffers (which must agree, so every byte is written), against the oracle (oracle/minecraft_api.py,
   pinned bit for bit to the reference's golden) and the golden itself.
   - Bit for bit where the arithmetic is restated: the upsampled climate planes and the smooth elevation (torch's two
     bilinear kernels), and the elevation without detail noise.
   - Three functions are not correctly rounded on either side: torch's CPU sqrt (the Sobel gradient), asin (the growing
     season) and pow(., 1.5) (the detail-noise amplitude); the device's are sqrt (correctly rounded), asinf and powf.
     Their bounds, from the functions' documented / measured errors:
       slope ratio  |d| <= 2^-21 |sr|  (torch sqrt <= 1 ulp, device 0.5 ulp; the division by pixel_size_m rounds once)
       growing season  |d| <= 2e-4 days  (asin: device <= 2 ulp, torch <= 6.3e-8 absolute; / 3.14159, 0.5 - ., x 365)
       eff tree moisture  |d| <= |tm| (2e-4 / 90 + 2^-22) + 2^-21 |eff|
       detail noise  |d| <= (|n_c| 100 + |n_f| 70) |noise| sf psm / nr 2^-16 + 2 ulp(elev)
     A biome id may differ only where its deciding quantity is within its bound of a cut-off (slope ratio against 0.62,
     0.78 and the bare threshold; growing season against 60; eff against 0.2, 0.5, 0.8, 1.3); an int16 elevation only
     where the fp32 value is within its bound of an integer; the fp32 elevation must lie within its bound.  The test
     reports how many pixels each case excused and fails on any other difference.
   NaN is compared by position (the GPU's canonical NaN has different sign and payload bits from x86's).
2. Every argument check of the entry point.
3. The pipeline: `get_minecraft` and `minecraft_payload` of a small TerrainPipeline against the oracle on `get()`'s
   output with the same injected noise, at scales 1, 2, 4 and 8, with the payload compared as bytes.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import minecraft_api as O
from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import TerrainPipeline
from terrain_diffusion_b200.inference import minecraft as M
from terrain_diffusion_b200.models import EDMUnet2D
from tests._igemm_ref import Guarded, report
from tests._minecraft_inputs import CASES, case_world, stand_in_noise
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
G = np.load(Path(__file__).resolve().parent / "golden" / "minecraft_golden.npz")
B_GS = 2e-4


@pytest.fixture(scope="module")
def excused(request):
    found: dict = {}
    yield found
    report(request.config, [f"{k}: {v}" for k, v in found.items()])


def assert_bits(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ at {int((np.isnan(got) ^ nan).sum())}"
    diff = (got.view(np.uint32) != want.view(np.uint32)) & ~nan
    if diff.any():
        i = tuple(int(v) for v in np.argwhere(diff)[0])
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ in their bits; first at {i}: got {got[i]!r}, "
                             f"want {want[i]!r}")


def planes_fn(i0, j0, h, w):
    return np.stack([stand_in_noise(c, i0, j0, h, w) for c in M.NOISE_CONFIGS])


def _int16_out(n, fill):
    raw = torch.full((n + 64,), 0x5A5A, dtype=torch.int16, device=DEV)
    body = raw[32:32 + n]
    body.fill_(fill)
    return raw, body


def run_kernel(win, centre, climate, noise, scale, oi, oj, H, W, noise_scale, psm, nr):
    """tdx_minecraft_readout through its C entry point: {'elev', 'elev_smooth', 'climate', 'biome', 'body'}."""
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, F32)).to(DEV)
    e, c, ctr, nz = dev(win), dev(climate), dev(centre), dev(noise)
    h, w = win.shape
    ptr = lambda t: None if t is None else t.data_ptr()
    detail = int(scale > 1 and noise_scale > 0)
    scal = (noise_scale * 100.0, noise_scale * 70.0, psm, nr, 40.0 * psm / 90.0)
    outs = {k: Guarded(s, torch.float32, DEV) for k, s in (("elev", (H, W)), ("elev_smooth", (H, W)),
                                                           ("climate", (5, H, W)))}
    if climate is None:
        outs["climate"] = None
    lib = L.lib()
    got = {}
    for fill in (0, -1):
        raw_b, biome = _int16_out(H * W, fill)
        raw_p, body = _int16_out(2 * H * W, fill)
        L.call(lib.tdx_minecraft_readout, DEV, e.data_ptr(), h, w, scale, oi, oj, ptr(ctr), ptr(c), ptr(nz), H, W,
               detail, *scal, outs["elev"].data_ptr(), outs["elev_smooth"].data_ptr(),
               ptr(outs["climate"]), biome.data_ptr(), None)
        L.call(lib.tdx_minecraft_readout, DEV, e.data_ptr(), h, w, scale, oi, oj, ptr(ctr), ptr(c), ptr(nz), H, W,
               detail, *scal, None, None, None, None, body.data_ptr())
        torch.cuda.synchronize()
        for raw, n in ((raw_b, H * W), (raw_p, 2 * H * W)):
            assert bool((raw[:32] == 0x5A5A).all()) and bool((raw[32 + n:] == 0x5A5A).all()), "int16 guard written"
        got.setdefault("biome", []).append(biome.cpu().numpy().reshape(H, W).copy())
        got.setdefault("body", []).append(body.cpu().numpy().tobytes())
    assert np.array_equal(*got["biome"]) and got["body"][0] == got["body"][1], "some int16 outputs were not written"
    res = {"biome": got["biome"][0], "body": got["body"][0]}
    for k, g in outs.items():
        if g is not None:
            g.check(k)
            res[k] = g.view.cpu().numpy()
    res["climate"] = res.get("climate")
    return res


def biome_excuse(v):
    """Pixels whose biome may differ: a deciding quantity within its bound of a cut-off (module docstring)."""
    with np.errstate(invalid="ignore"):
        sr, bt = v["slope_ratio"].astype(np.float64), v["bare_threshold"].astype(np.float64)
        b_sr = 2.0 ** -21 * np.abs(sr)
        near = (np.abs(sr - F32(0.62)) <= b_sr) | (np.abs(sr - F32(0.78)) <= b_sr) | (np.abs(sr - bt) <= b_sr)
        gs = v["growing_season"].astype(np.float64)
        near |= np.abs(gs - 60.0) <= B_GS
        tm, eff = v["tree_moisture"].astype(np.float64), v["eff"].astype(np.float64)
        b_eff = np.abs(tm) * (B_GS / 90.0 + 2.0 ** -22) + 2.0 ** -21 * np.abs(eff)
        for c in (0.2, 0.5, 0.8, 1.3):
            near |= np.abs(eff - F32(c)) <= b_eff
    return near


def elev_bound(r, noise, noise_scale, psm, nr):
    """Per-pixel bound on the detail-noised elevation (0 where the arithmetic is restated exactly)."""
    sm = r["elev_smooth"].astype(np.float64)
    if noise_scale <= 0 or r["scale"] == 1:
        return np.zeros_like(sm)
    g = r["vars_gradient"].astype(np.float64)
    with np.errstate(invalid="ignore"):
        sf = np.clip(g / (40.0 * psm / 90.0), 0.0, 1.0) ** 1.5
        mag = (np.abs(noise[3]) * 100.0 + np.abs(noise[4]) * 70.0) * abs(noise_scale) * sf * psm / nr
        b = mag * 2.0 ** -16 + 2.0 * np.spacing(np.abs(r["elev"]).astype(F32)).astype(np.float64)
    return np.where(sm >= 0, b, 0.0)


def compare(got, r, noise, noise_scale, psm, nr, what, excused):
    """The device outputs against the oracle `r` under the rules of the module docstring; returns the counts."""
    assert_bits(got["elev_smooth"], r["elev_smooth"], what + " elev_smooth")
    if r["climate"] is not None:
        assert_bits(got["climate"], r["climate"], what + " climate")
    bound = elev_bound(r, noise, noise_scale, psm, nr)
    want_e = r["elev"].astype(np.float64)
    nan = np.isnan(want_e)
    assert np.array_equal(np.isnan(got["elev"]), nan), what + " elev NaN positions"
    exact = bound == 0
    assert_bits(np.where(exact, got["elev"], 0), np.where(exact, r["elev"], 0), what + " elev (restated exactly)")
    with np.errstate(invalid="ignore"):
        err = np.abs(got["elev"].astype(np.float64) - want_e)
        inside = (err <= bound) | nan | (got["elev"] == r["elev"])            # equal infinities have a NaN difference
    assert np.all(inside), f"{what}: elev outside its bound by {np.nanmax(np.where(inside, 0, err - bound)):.3g}"
    fp32_diff = int(((got["elev"] != r["elev"]) & ~nan).sum())
    H, W = r["elev"].shape
    e16_got = np.frombuffer(got["body"], "<i2", count=H * W).reshape(H, W)
    e16_want = np.frombuffer(r["body"], "<i2", count=H * W).reshape(H, W)
    with np.errstate(invalid="ignore"):
        near_int = np.minimum(want_e - np.floor(want_e), np.ceil(want_e) - want_e) <= bound
    bad16 = (e16_got != e16_want)
    assert not (bad16 & ~near_int).any(), f"{what}: int16 elevation differs at {int((bad16 & ~near_int).sum())} pixels"
    assert np.array_equal(np.frombuffer(got["body"], "<i2", offset=2 * H * W).reshape(H, W), got["biome"])
    badb = got["biome"] != r["biome"]
    if r["vars"] is not None:
        ok = biome_excuse(r["vars"])
        assert not (badb & ~ok).any(), (f"{what}: biome differs at {int((badb & ~ok).sum())} pixels outside the "
                                        f"excused set; first at {tuple(np.argwhere(badb & ~ok)[0])}")
    else:
        assert not badb.any(), what + " biome (no climate: plains)"
    excused[what] = (f"biome ids excused {int(badb.sum())} (of {int(biome_excuse(r['vars']).sum()) if r['vars'] else 0}"
                     f" pixels near a cut-off), int16 elevations excused {int(bad16.sum())}, fp32 elevations within "
                     f"their bound but not equal {fp32_diff}")


def case_inputs(name):
    world, (i1, j1, i2, j2, scale, noise) = case_world(name)
    H, W = i2 - i1, j2 - j1
    nr = world.native_resolution
    wi1, wj1, wi2, wj2, oi, oj = O.minecraft_window(i1, j1, i2, j2, scale)
    nz = planes_fn(i1, j1, H, W)
    if scale == 1:
        win = world.get_np(wi1, wj1, wi2, wj2, False)["elev"]
        out = world.get_np(i1, j1, i2, j2, True)
        return dict(win=win, centre=out["elev"], climate=out["climate"], noise=nz, scale=1, oi=1, oj=1, H=H, W=W,
                    noise_scale=noise, psm=nr, nr=nr)
    out = world.get_np(wi1, wj1, wi2, wj2, True)
    return dict(win=out["elev"], centre=None, climate=out["climate"], noise=nz, scale=scale, oi=oi, oj=oj, H=H, W=W,
                noise_scale=noise, psm=nr / scale, nr=nr)


def oracle_of(a):
    r = O.readout(a["win"], a["climate"], a["noise"], a["scale"], a["oi"], a["oj"], a["H"], a["W"], a["noise_scale"],
                  a["psm"], a["nr"], centre=a["centre"])
    r["body"] = O.payload(r["elev"], r["biome"])
    r["scale"] = a["scale"]
    r["vars_gradient"] = (r["vars"] or {}).get("gradient", O.gradient(
        O.upsample_crop(a["win"], a["scale"], a["oi"] - 1, a["oj"] - 1, a["H"] + 2, a["W"] + 2)))
    return r


@pytest.mark.parametrize("name", list(CASES))
def test_kernel_matches_oracle_and_golden(name, excused):
    a = case_inputs(name)
    r = oracle_of(a)
    got = run_kernel(a["win"], a["centre"], a["climate"], a["noise"], a["scale"], a["oi"], a["oj"], a["H"], a["W"],
                     a["noise_scale"], a["psm"], a["nr"])
    compare(got, r, a["noise"], a["noise_scale"], a["psm"], a["nr"], name, excused)
    if f"{name}.error" in G or f"{name}.body" not in G:
        return
    # the oracle is the golden on the host that recorded it (tests/test_minecraft_cpu.py: every array by its digest,
    # small cases element by element); check the device against the golden's body and stored arrays too, under the
    # same rules
    g = dict(r)
    if f"{name}.elev" in G:
        g["elev"] = G[f"{name}.elev"]
    g["body"] = G[f"{name}.body"].tobytes()
    H, W = a["H"], a["W"]
    g["biome"] = np.frombuffer(g["body"], "<i2", offset=2 * H * W).reshape(H, W)
    if f"{name}.climate" in G:
        g["climate"], g["elev_smooth"] = G[f"{name}.climate"], G[f"{name}.elev_smooth"]
    compare(got, g, a["noise"], a["noise_scale"], a["psm"], a["nr"], name + " vs golden", excused)


@pytest.mark.parametrize("scale", [1, 2, 3, 8])
def test_kernel_random_windows_with_specials(scale, excused):
    """Random native windows with NaN / +-inf elevation and NaN climate, crops whose pixel counts sit on either side of
    the 16-pixel gemm blocks and the 20480-element oneDNN switch, noise on, off and negative."""
    rng = np.random.RandomState(scale)
    for H, W, ns in ((1, 1, 1.0), (1, 17, 1.0), (5, 7, 0.0), (16, 16, -1.0), (13, 29, 1.0), (141, 141, 1.0),
                     (142, 142, 2.5), (30, 1, 1.0)):
        if scale == 1:
            h, w, oi, oj = H + 2, W + 2, 1, 1
        else:
            h, w = -(-H // scale) + 5, -(-W // scale) + 5
            oi, oj = 2 * scale + int(rng.randint(0, scale)), 2 * scale + int(rng.randint(0, scale))
        win = (rng.randn(h, w) * 800 + 300).astype(F32)
        clim = np.stack([rng.uniform(-25, 35, (h, w)), rng.uniform(0, 1500, (h, w)), rng.uniform(0, 4000, (h, w)),
                         rng.uniform(0, 150, (h, w)), rng.uniform(-0.006, 0.006, (h, w))]).astype(F32)
        win.ravel()[rng.randint(0, h * w, 3)] = (np.nan, np.inf, -np.inf)
        clim[0].ravel()[rng.randint(0, h * w)] = np.nan
        centre = None
        if scale == 1:
            centre = win[1:-1, 1:-1].copy()
            clim = clim[:, 1:-1, 1:-1].copy()
        noise = rng.uniform(-1, 1, (5, H, W)).astype(F32)
        nr = 90.0
        psm = nr / scale if scale > 1 else nr
        a = dict(win=win, centre=centre, climate=clim, noise=noise, scale=scale, oi=oi, oj=oj, H=H, W=W,
                 noise_scale=ns, psm=psm, nr=nr)
        with np.errstate(invalid="ignore", over="ignore"):
            r = oracle_of(a)
        got = run_kernel(win, centre, clim, noise, scale, oi, oj, H, W, ns, psm, nr)
        compare(got, r, noise, ns, psm, nr, f"random x{scale} {H}x{W} noise {ns}", excused)
        got2 = run_kernel(win, centre, None, noise, scale, oi, oj, H, W, ns, psm, nr)       # no climate: plains
        assert (got2["biome"] == 1).all() and got2["climate"] is None
        assert_bits(got2["elev_smooth"], got["elev_smooth"], "without climate")
        assert_bits(got2["elev"], got["elev"], "without climate")


def test_argument_checks():
    x = torch.zeros(6, 8, 8, device=DEV)
    n = torch.zeros(5, 4, 4, device=DEV)
    p, q = x.data_ptr(), n.data_ptr()
    lib = L.lib()
    s = (1.0, 1.0, 45.0, 90.0, 20.0)
    ok = (p, 8, 8, 2, 5, 5, None, p, q, 4, 4, 1, *s, p, None, None, None, None)
    L.call(lib.tdx_minecraft_readout, DEV, *ok)                     # the baseline call is accepted
    torch.cuda.synchronize()

    def with_(**kw):
        names = ("elev h w scale oi oj centre climate noise H W detail amp_c amp_f psm nr div elev_out smooth_out "
                 "climate_out biome_out payload").split()
        args = dict(zip(names, ok))
        args.update(kw)
        return tuple(args[k] for k in names)

    for bad in [with_(elev=None), with_(elev_out=None),                              # no input / no output
                with_(climate=None, climate_out=p),                                  # climate_out without climate
                with_(noise=None), with_(noise=None, climate=None),                  # noise needed (climate, detail)
                with_(payload=p + 1), with_(biome_out=p + 1),                        # odd int16 addresses
                with_(scale=0), with_(h=2), with_(H=0), with_(W=0), with_(H=70000),  # shapes
                with_(oi=0), with_(oj=0), with_(oi=12), with_(oj=12),                # crop and its ring outside
                with_(centre=p),                                                     # centre at scale 2
                with_(scale=1, h=6, w=6, oi=1, oj=1, detail=0),                      # scale 1 without centre
                with_(scale=1, h=6, w=6, oi=1, oj=1, centre=p, detail=1),            # scale 1 with detail noise
                with_(scale=1, h=6, w=7, oi=1, oj=1, centre=p, detail=0),            # scale 1 window not [H+2][W+2]
                with_(scale=1, h=6, w=6, oi=2, oj=1, centre=p, detail=0, H=3)]:      # scale 1 crop not at (1, 1)
        with pytest.raises(L.TdxError):
            L.call(lib.tdx_minecraft_readout, DEV, *bad)
    L.call(lib.tdx_minecraft_readout, DEV, *with_(scale=1, h=6, w=6, oi=1, oj=1, centre=p, detail=0))
    L.call(lib.tdx_minecraft_readout, DEV, *with_(noise=None, climate=None, detail=0))
    torch.cuda.synchronize()


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


WINDOWS = [(-20, 10, 44, 90), (-37, -5, -21, 11), (3, -77, 4, 60), (-130, 7, 70, 8), (0, 0, 16, 16), (5, 5, 6, 6)]


@pytest.mark.parametrize("scale", [1, 2, 4, 8])
def test_pipeline_against_oracle(pipe, scale, excused):
    calls = []

    def noise_fn(cfg, i0, j0, h, w):
        calls.append(cfg)
        return stand_in_noise(cfg, i0, j0, h, w)

    def get_np(a, b, c, d, with_climate=True):
        out = pipe.get(a, b, c, d, with_climate)
        return {k: (None if v is None else v.cpu().numpy()) for k, v in out.items()}

    for win in WINDOWS:
        for noise in ((1.0, 0.0) if scale > 1 else (1.0,)):
            r = O.request(get_np, *win, scale, noise, pipe.native_resolution, planes_fn)
            r["scale"] = scale
            ring = O.minecraft_window(*win, scale)
            if scale == 1:
                xp = get_np(*ring[:4], False)["elev"]
            else:
                h = get_np(*ring[:4], False)["elev"]
                xp = O.upsample_crop(h, scale, ring[4] - 1, ring[5] - 1, win[2] - win[0] + 2, win[3] - win[1] + 2)
            r["vars_gradient"] = O.gradient(xp)
            calls.clear()
            out = pipe.get_minecraft(*win, scale=scale, noise=noise, noise_fn=noise_fn)
            assert len(calls) == len(set(calls)) == (5 if scale > 1 and noise > 0 else 3)
            assert all(v.is_cuda for v in (out["elev"], out["elev_smooth"], out["climate"], out["biome"]))
            body, hw = pipe.minecraft_payload(*win, scale=scale, noise=noise, noise_fn=noise_fn)
            assert hw == (win[2] - win[0], win[3] - win[1])
            got = {k: out[k].cpu().numpy() for k in ("elev", "elev_smooth", "climate", "biome")}
            got["body"] = body
            assert body == O.payload(got["elev"], got["biome"]), "payload is not the packing of get_minecraft's output"
            psm = pipe.native_resolution / scale if scale > 1 else pipe.native_resolution
            nz = planes_fn(win[0], win[1], *hw)
            compare(got, r, nz, noise, psm, pipe.native_resolution, f"pipeline x{scale} {win} noise {noise}", excused)
            if not (got["biome"] != r["biome"]).any() and np.array_equal(
                    np.frombuffer(body, "<i2", count=hw[0] * hw[1]),
                    np.frombuffer(r["body"], "<i2", count=hw[0] * hw[1])):
                assert body == r["body"]
    pipe._host_views = True                                    # WorldPipeline: CPU tensors through pinned copies
    try:
        out = pipe.get_minecraft(*WINDOWS[0], scale=scale, noise_fn=stand_in_noise)
    finally:
        pipe._host_views = False
    assert not out["elev"].is_cuda and out["elev"].is_pinned() and out["biome"].dtype == torch.int16
