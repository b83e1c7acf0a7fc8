"""Terrain API read-out on the GPU (csrc/tdx_post.cu `tdx_terrain_upsample`, `WorldPipeline.get_terrain` /
`terrain_payload`).

1. The C entry point, every output in a guarded buffer (fp32 planes NaN-filled; the byte payload written twice over
   0x00- and 0xFF-filled buffers, which must agree, so every byte is written), compared
   (a) bit for bit with the oracle (oracle/terrain_api.py `upsample_crop`, pinned to the reference's golden) and with live
       torch CPU `F.interpolate` on this host: torch has two CPU kernels and picks by the size of the whole upsampled
       window, so native windows 3..24 and 64..300 on both axes at scales 2..8 and 16 cover both; every crop offset
       0..scale-1 on both axes, 1x1, 1xN, Nx1 and 16x16 crops, NaN / +-inf in the window and both int16 clip edges.
       NaN must be NaN in the same positions (its sign and payload are the producer's, and differ between x86 and the
       GPU); every other value is compared by its bits.
   (b) against fp64 bilinear interpolation with torch's own fp32 weights (the weights are part of torch's definition,
       not an error): |got - ref| <= gamma_n * sum|w_ab x_ab|, n = the rounded operations on the longest path: 4 for the
       separable kernel (wl1*x01, fma -> t, hl1*t1, fma) and 5 for the per-pixel-weight kernel (hl0*wl1, w01*x01, three
       fma).  The worst share of each bound is written to the terminal.
2. The pipeline: `get_terrain` and `terrain_payload` of a small TerrainPipeline against `_get_terrain` /
   `_binary_response` restated on `get()`'s CPU output with live torch, for negative and unaligned windows at scales
   1, 2, 4 and 8; the payload is compared as bytes.
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import terrain_api as O
from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import TerrainPipeline
from terrain_diffusion_b200.models import EDMUnet2D
from tests._igemm_ref import Guarded, report
from tests._terrain_api_inputs import CASES, case_world, planes
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
G = np.load(Path(__file__).resolve().parent / "golden" / "terrain_api_golden.npz")
U = 2.0 ** -24


def gamma(n: int) -> float:
    return n * U / (1.0 - n * U)


@pytest.fixture(scope="module")
def margins(request):
    found: dict = {}
    yield found
    report(request.config, [f"worst {kind}: {v:.3g} of the bound" for kind, v in sorted(found.items())])


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


def run_kernel(native: np.ndarray, scale: int, oi: int, oj: int, H: int, W: int, with_climate: bool = True):
    """tdx_terrain_upsample on native [6, h, w] (elevation + 5 climate planes): (elev [H, W], climate [5, H, W] | None,
    payload bytes), each from guarded buffers."""
    x = torch.from_numpy(np.ascontiguousarray(native, F32)).to(DEV)
    h, w = native.shape[-2:]
    clim = x[1:] if with_climate else None
    e_out = Guarded((H, W), torch.float32, DEV)
    c_out = Guarded((5, H, W), torch.float32, DEV) if with_climate else None
    L.call(L.lib().tdx_terrain_upsample, DEV, x[0].data_ptr(), clim.data_ptr() if with_climate else None, h, w, scale,
           oi, oj, H, W, e_out.data_ptr(), c_out.data_ptr() if with_climate else None, None)
    nbytes = H * W * (18 if with_climate else 2)
    bodies = []
    for fill in (0x00, 0xFF):
        raw = torch.full((nbytes + 128,), 0x5A, dtype=torch.uint8, device=DEV)
        body = raw[64:64 + nbytes]
        body.fill_(fill)
        L.call(L.lib().tdx_terrain_upsample, DEV, x[0].data_ptr(), clim.data_ptr() if with_climate else None, h, w,
               scale, oi, oj, H, W, None, None, body.data_ptr())
        torch.cuda.synchronize()
        guards = torch.cat([raw[:64], raw[64 + nbytes:]])
        assert bool((guards == 0x5A).all()), "payload: written outside the buffer"
        bodies.append(body.cpu().numpy().tobytes())
    assert bodies[0] == bodies[1], "payload: some bytes were not written"
    torch.cuda.synchronize()
    e_out.check("elev_out")
    if with_climate:
        c_out.check("climate_out")
    return e_out.view.cpu().numpy(), c_out.view.cpu().numpy() if with_climate else None, bodies[0]


def check_payload(body: bytes, elev, climate, what):
    """The wire body against the restated packing: int16 exact, the fp32 climate by bits with NaN by position."""
    H, W = elev.shape
    want = O.terrain_payload(elev, climate)
    assert len(body) == len(want), what
    assert body[:2 * H * W] == want[:2 * H * W], f"{what}: int16 elevation differs"
    if climate is not None:
        got_c = np.frombuffer(body, "<f4", offset=2 * H * W).reshape(H, W, 4)
        assert_bits(got_c, np.transpose(climate[:4], (1, 2, 0)), f"{what}: climate payload")


def fp64_check(native, scale, oi, oj, H, W, got, margins):
    h, w = native.shape[-2:]
    hi0, hi1, hl0, hl1 = O.upsample_taps(h, scale, np.arange(oi, oi + H))
    wi0, wi1, wl0, wl1 = O.upsample_taps(w, scale, np.arange(oj, oj + W))
    x = native.astype(np.float64)
    terms = [hl[:, None].astype(np.float64) * wl[None, :].astype(np.float64) * x[:, hi[:, None], wi[None, :]]
             for hl, hi in ((hl0, hi0), (hl1, hi1)) for wl, wi in ((wl0, wi0), (wl1, wi1))]
    ref = sum(terms)
    small = (h + w) * scale <= 128
    kind = "small kernel" if small else "separable kernel"
    bound = gamma(5 if small else 4) * sum(np.abs(t) for t in terms)
    err = np.abs(got.astype(np.float64) - ref)
    assert np.all(err <= bound), f"{kind} x{scale} {h}x{w}: outside the fp64 bound by {float((err - bound).max()):.3g}"
    share = float((err / np.where(bound > 0, bound, 1.0)).max())
    margins[kind] = max(margins.get(kind, 0.0), share)


def torch_crop(native, scale, oi, oj, H, W):
    full = F.interpolate(torch.from_numpy(native)[None], scale_factor=scale, mode="bilinear", align_corners=False)[0]
    return full[:, oi:oi + H, oj:oj + W].numpy()


def crops(h, w, scale, rng):
    """(oi, oj, H, W): every offset 0..scale-1 on each axis, with full-width, 1-pixel and 16-pixel extents."""
    Hs, Ws = h * scale, w * scale
    out = []
    for k in range(scale):
        oi, oj = k, (3 * k + 1) % scale
        kind = k % 4
        H = {0: Hs - oi, 1: 1, 2: min(16, Hs - oi), 3: Hs - oi - int(rng.randint(0, scale))}[kind]
        W = {0: Ws - oj, 1: Ws - oj, 2: min(16, Ws - oj), 3: 1}[kind]
        out.append((oi, oj, max(H, 1), max(W, 1)))
    out.append((Hs - 1, Ws - 1, 1, 1))
    return out


SHAPES = [(3, w) for w in range(3, 25)] + [(h, 3) for h in range(4, 25)] + \
         [(3, 64), (64, 3), (5, 100), (130, 6), (3, 300), (300, 4), (20, 70), (8, 8), (16, 16)]


@pytest.mark.parametrize("scale", [2, 3, 4, 5, 6, 7, 8, 16])
def test_kernel_bit_exact_and_fp64(scale, margins):
    rng = np.random.RandomState(100 + scale)
    paths = set()
    for h, w in SHAPES:
        native = planes(scale * 1000 + h * 31 + w, -h // 2, 7, h - h // 2, 7 + w)   # some rows past the clip edges
        ref_full = torch_crop(native, scale, 0, 0, h * scale, w * scale)
        paths.add((h + w) * scale <= 128)
        for oi, oj, H, W in crops(h, w, scale, rng):
            e, c, body = run_kernel(native, scale, oi, oj, H, W)
            want = O.upsample_crop(native, scale, oi, oj, H, W)
            what = f"x{scale} native {h}x{w} crop {H}x{W} at ({oi},{oj})"
            assert_bits(e, want[0], what + " elev vs oracle")
            assert_bits(c, want[1:], what + " climate vs oracle")
            live = ref_full[:, oi:oi + H, oj:oj + W]
            assert_bits(np.concatenate([e[None], c]), live, what + " vs live torch")
            check_payload(body, e, c, what)
            fp64_check(native, scale, oi, oj, H, W, np.concatenate([e[None], c]), margins)
    assert paths == {True, False}


@pytest.mark.parametrize("scale", [1, 2, 3, 8, 16])
def test_kernel_nan_inf_and_clip_edges(scale):
    rng = np.random.RandomState(scale)
    for h, w in ((3, 3), (4, 11), (3, 40), (25, 7), (6, 60)):
        native = planes(77 + scale, 0, 0, h, w, specials=True)
        native[1, 0, 0], native[2, h - 1, w - 1] = np.inf, np.nan          # specials in the climate too
        native[0, 1, :2] = (32767.5, -32768.25)
        native[0, h - 1, -1] = 40000.0
        Hs, Ws = h * scale, w * scale
        for oi, oj, H, W in [(0, 0, Hs, Ws), (Hs - 1, 0, 1, Ws), (0, Ws - 1, Hs, 1)] + \
                [(int(rng.randint(0, Hs)), int(rng.randint(0, Ws)), 1, 1)]:
            with np.errstate(invalid="ignore"):
                want = O.upsample_crop(native, scale, oi, oj, H, W)
            e, c, body = run_kernel(native, scale, oi, oj, H, W)
            what = f"x{scale} {h}x{w} specials crop {H}x{W} at ({oi},{oj})"
            assert_bits(e, want[0], what)
            assert_bits(c, want[1:], what)
            if scale > 1:
                assert_bits(np.concatenate([e[None], c]), torch_crop(native, scale, oi, oj, H, W), what + " vs torch")
            check_payload(body, e, c, what)
            e2, c2, body2 = run_kernel(native, scale, oi, oj, H, W, with_climate=False)
            assert c2 is None and len(body2) == 2 * H * W and body2 == body[:2 * H * W]
            assert_bits(e2, e, what + " without climate")
    if scale == 1:                         # a plain copy: inf stays inf, nothing turns into NaN
        native = planes(5, 0, 0, 4, 4, specials=True)
        e, c, _ = run_kernel(native, 1, 0, 0, 4, 4)
        assert_bits(e, native[0], "scale 1 copy")
        assert_bits(c, native[1:], "scale 1 copy climate")
    e16 = np.frombuffer(run_kernel(np.stack([np.array([[np.nan, np.inf, -np.inf], [32767.9, -32768.0, -32768.5],
                                                        [-0.5, -0.0, 0.99]], F32)] * 6), 1, 0, 0, 3, 3)[2][:18], "<i2")
    assert e16.tolist() == [0, 32767, -32768, 32767, -32768, -32768, -1, 0, 0]


@pytest.mark.parametrize("name", list(CASES))
def test_kernel_matches_reference_golden(name):
    world, (i1, j1, i2, j2, scale) = case_world(name)
    ni1, nj1, ni2, nj2, oi, oj = O.terrain_window(i1, j1, i2, j2, scale)
    native = planes(world.seed, ni1, nj1, ni2, nj2, world.specials)
    e, c, body = run_kernel(native, scale, oi, oj, i2 - i1, j2 - j1)
    assert_bits(e, G[f"{name}.elev"], name)
    assert_bits(c, G[f"{name}.climate"], name)
    assert body == G[f"{name}.body"].tobytes()


def test_argument_checks():
    x = torch.zeros(6, 4, 4, device=DEV)
    lib = L.lib()
    p = x.data_ptr()
    for args in [(p, None, 4, 4, 0, 0, 0, 4, 4, p, None, None),           # scale 0
                 (p, None, 4, 4, 2, 1, 0, 8, 4, p, None, None),           # crop past the upsampled window
                 (p, None, 4, 4, 2, -1, 0, 4, 4, p, None, None),
                 (p, None, 4, 4, 2, 0, 0, 4, 4, None, None, None),        # no output
                 (p, None, 4, 4, 2, 0, 0, 4, 4, None, p, None),           # climate out without climate
                 (p, p, 4, 4, 2, 0, 0, 4, 4, None, None, p + 1)]:         # odd payload address
        with pytest.raises(L.TdxError):
            L.call(lib.tdx_terrain_upsample, DEV, *args)


# ------------------------------------------------------------------------------------------------------ pipeline
def ref_get_terrain(get, i1, j1, i2, j2, scale):
    """api.py _get_terrain restated on a get() returning CPU tensors."""
    if scale == 1:
        out = get(i1, j1, i2, j2)
        return out["elev"], out["climate"]
    ni1, nj1, ni2, nj2 = i1 // scale, j1 // scale, -(-i2 // scale), -(-j2 // scale)
    out = get(ni1 - 1, nj1 - 1, ni2 + 1, nj2 + 1)
    ci, cj = scale + i1 - ni1 * scale, scale + j1 - nj1 * scale
    e = F.interpolate(out["elev"][None, None], scale_factor=scale, mode="bilinear", align_corners=False).squeeze()
    c = F.interpolate(out["climate"][None], scale_factor=scale, mode="bilinear", align_corners=False).squeeze(0)
    return e[ci:ci + i2 - i1, cj:cj + j2 - j1], c[:, ci:ci + i2 - i1, cj:cj + j2 - j1]


def ref_body(elev, climate) -> bytes:
    """api.py _binary_response's body restated: numpy floor / clip / '<i2', then climate[:4] as HWC '<f4'."""
    e16 = np.clip(np.floor(elev.numpy().astype(F32, copy=False)), -32768, 32767).astype("<i2", copy=False)
    return e16.tobytes() + np.transpose(climate[:4].numpy().astype("<f4", copy=False), (1, 2, 0)).tobytes()


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


WINDOWS = [(-20, 10, 44, 90), (-37, -5, -21, 11), (3, -77, 4, 60), (-130, 7, 70, 8), (0, 0, 16, 16)]


@pytest.mark.parametrize("scale", [1, 2, 4, 8])
def test_pipeline_against_reference_functions(pipe, scale):
    def get_cpu(a, b, c, d):
        out = pipe.get(a, b, c, d)
        return {k: v.cpu() for k, v in out.items()}

    for win in WINDOWS:
        e_ref, c_ref = ref_get_terrain(get_cpu, *win, scale)
        out = pipe.get_terrain(*win, scale=scale)
        assert out["elev"].is_cuda and out["climate"].is_cuda
        assert_bits(out["elev"].cpu().numpy(), e_ref.numpy(), f"get_terrain elev x{scale} {win}")
        assert_bits(out["climate"].cpu().numpy(), c_ref.numpy(), f"get_terrain climate x{scale} {win}")
        assert pipe.get_terrain(*win, scale=scale, with_climate=False)["climate"] is None
        body, hw = pipe.terrain_payload(*win, scale=scale)
        assert hw == (win[2] - win[0], win[3] - win[1])
        assert body == ref_body(e_ref, c_ref), f"payload x{scale} {win}"
    pipe._host_views = True                                    # WorldPipeline: CPU tensors through one pinned copy
    try:
        out = pipe.get_terrain(*WINDOWS[0], scale=scale)
    finally:
        pipe._host_views = False
    assert not out["elev"].is_cuda and out["elev"].is_pinned()
    e_ref, c_ref = ref_get_terrain(get_cpu, *WINDOWS[0], scale)
    assert_bits(out["elev"].numpy(), e_ref.numpy(), "host elev")
    assert_bits(out["climate"].numpy(), c_ref.numpy(), "host climate")


def test_host_torch_dispatch_is_the_goldens():
    """Report (not hide) a torch CPU build that dispatches differently from the one that recorded the golden: the live
    comparisons above would then be the ones to fail."""
    cap = torch.backends.cpu.get_cpu_capability()
    print(f"\ntorch {torch.__version__} CPU capability {cap}; golden recorded with torch {G['torch_version']} "
          f"{G['cpu_capability']}")
