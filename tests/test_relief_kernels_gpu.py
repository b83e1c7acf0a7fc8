"""The three shaded-relief kernels of csrc/tdx_relief.cu, each through its C entry point, on every branch and at the sizes
the explorer renders:

  tdx_relief_stats     NaN count and the bit patterns of nanmin / nanmax of max(0, x), exactly, at sizes around the
                       grid cap (4 x SMs x 256 elements, read from this device) with the special values both in the first
                       grid pass and past it; the stats buffer starts as garbage, so the call must zero it;
  tdx_relief_gaussian  bit for bit against scipy.ndimage.gaussian_filter of the NaN-filled plane, including the
                       one-tap filter, radius 96 on images the reflection wraps several times, and 4096^2; every
                       argument error returns before any launch;
  tdx_relief_shade     bit for bit against the kernel's contract (tests/_relief_contract.py) except the pixels it
                       excuses (fp64 transcendentals near an fp32 rounding midpoint), and every pixel against the
                       oracle under the rule of tests/test_relief_gpu.py.

The benchmark field of tools/bench_relief.py is also run through get_relief_map at 512^2 and 1024^2.  Every output lives
in a guarded buffer (tests/_igemm_ref.Guarded): a write outside it fails, and so does an element left unwritten.  The
excused pixels, the worst share of the 2e-5 bound and the benchmark's worst pixel are written to the terminal."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter

from oracle import relief as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import get_relief_map
from terrain_diffusion_b200.inference.relief import gaussian_taps
from tests import _relief_contract as K
from tests._igemm_ref import Guarded, device_sm_count, report
from tests._post_inputs import field
from tests._relief_inputs import bench_field

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
GARBAGE = -0x21524111          # 0xDEADBEEF: above every ~bits(nanmin) a zeroed buffer could hold
UNWRITTEN = 3.0                # the shade kernel never writes a value above 1 (NaN is a legal output, so not NaN)


@pytest.fixture(scope="module")
def notes(request):
    """Lines written to the terminal (also under -q) when the module is done."""
    found: list = []
    yield found
    report(request.config, found)


def dev(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).to(DEV)


def fetch(g: Guarded, what: str) -> np.ndarray:
    torch.cuda.synchronize()
    g.check(what)
    return g.view.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------- stats

def grid_cap() -> int:
    """Elements one pass of tdx_relief_stats' grid covers: 4 blocks per SM of 256 threads."""
    return 4 * device_sm_count() * 256


def run_stats(x: np.ndarray) -> np.ndarray:
    """tdx_relief_stats of x into a garbage-filled guarded buffer; the input is followed by NaN, so a read past n
    changes the count."""
    n = x.size
    buf = torch.full((n + 64,), float("nan"), dtype=torch.float32, device=DEV)
    buf[:n] = dev(x.reshape(-1))
    g = Guarded((3,), torch.float32, DEV)
    g.view.view(torch.int32).fill_(GARBAGE)
    L.call(L.lib().tdx_relief_stats, DEV, buf.data_ptr(), n, g.data_ptr())
    return fetch(g, f"stats n={n}").view(np.uint32)


SPECIALS = {"nan": np.nan, "-0": -0.0, "+0": 0.0, "negative": -3.25, "+inf": np.inf, "-inf": -np.inf,
            "subnormal": np.float32(1e-45), "-subnormal": -np.float32(1e-45), "largest": np.finfo(F32).max}
SIZES = ["1", "31", "32", "255", "257", "cap-1", "cap+1", "1024^2", "4096^2"]


def stats_size(label: str, cap: int) -> int:
    if label.startswith("cap"):
        return cap + int(label[3:])
    if "^" in label:
        return int(label.split("^")[0]) ** 2
    return int(label)


def stats_inputs(n: int, cap: int):
    """(label, x): positive finite background (so a special value decides the extremum it touches) with each special
    value once in the first 256 elements and, when the array is longer than one grid pass, once past it; then all
    NaN and all <= 0."""
    rng = np.random.RandomState(n % 100003)
    base = rng.uniform(1.0, 1000.0, n).astype(F32)
    yield "background", base
    spots = [("first pass", (n - 1) // 2 if n <= 256 else 137)]
    if n > cap:
        spots.append(("past the grid cap", n - 1))
    for where, p in spots:
        for name, v in SPECIALS.items():
            x = base.copy()
            x[p] = v
            yield f"{name} at {p} ({where})", x
    yield "all NaN", np.full(n, np.nan, F32)
    x = -rng.uniform(0.0, 50.0, n).astype(F32)
    x[::3] = -0.0
    x[1::5] = 0.0
    x[n // 2] = -np.inf
    yield "all <= 0", x


@pytest.mark.parametrize("size", SIZES)
def test_stats_counts_and_extrema_exactly(size, notes):
    cap = grid_cap()
    n = stats_size(size, cap)
    beyond = 0
    for what, x in stats_inputs(n, cap):
        got = run_stats(x)
        want = K.encode_stats(x)
        assert np.array_equal(got, want), (size, what, [hex(v) for v in got], [hex(v) for v in want])
        assert int(got[0]) == int(np.isnan(x).sum()), (size, what)
        lo, hi = K.decode_stats(got)
        if np.isnan(x).all():
            assert K.is_fallback(lo, hi), (size, what)
            continue
        land = np.maximum(F32(0), x)
        with np.errstate(invalid="ignore"):
            want_lo, want_hi = np.nanmin(land) + F32(0), np.nanmax(land) + F32(0)   # + 0 turns numpy's -0 into +0
        assert np.array_equal(np.array([lo, hi], F32).view(np.uint32),
                              np.array([want_lo, want_hi], F32).view(np.uint32)), (size, what, lo, hi, want_lo, want_hi)
        beyond += "past the grid cap" in what
    if size == "cap+1":
        assert beyond == len(SPECIALS)
    notes.append(f"relief_stats n={n} ({size}, grid cap {cap}): exact; {beyond} cases with the special value past the "
                 "first grid pass")


# ------------------------------------------------------------------------------------------------------------- gaussian

def taps_of(sigmas):
    taps = [gaussian_taps(s) for s in sigmas]
    return np.ascontiguousarray(np.concatenate(taps), dtype=np.float64), [len(t) // 2 for t in taps]


def gaussian_call(xd, h, w, replace_nan, fill, n_sigma, w64, radius, tmp_ptr, out_ptr) -> int:
    """tdx_relief_gaussian called directly: returns its status code."""
    r32 = (C.c_int32 * max(1, len(radius)))(*radius)
    return L.lib().tdx_relief_gaussian(xd, h, w, replace_nan, fill, n_sigma, w64.ctypes.data_as(C.POINTER(C.c_double)),
                                       r32, tmp_ptr, out_ptr, L.current_stream_ptr(DEV))


def run_gaussian(x: np.ndarray, sigmas, fill=None) -> np.ndarray:
    h, w = x.shape
    xd = dev(x)
    w64, radius = taps_of(sigmas)
    tmp = Guarded((len(sigmas), h, w), torch.float32, DEV)
    out = Guarded((len(sigmas), h, w), torch.float32, DEV)
    rc = gaussian_call(xd.data_ptr(), h, w, int(fill is not None), 0.0 if fill is None else float(fill), len(sigmas),
                       w64, radius, tmp.data_ptr(), out.data_ptr())
    L.check(rc)
    fetch(tmp, "gaussian tmp")
    return fetch(out, "gaussian out")


def assert_scipy_bits(got, x, sigmas, fill, what):
    src = x if fill is None else np.where(np.isnan(x), F32(fill), x)
    for i, s in enumerate(sigmas):
        want = gaussian_filter(src, s)
        assert not np.isnan(got[i]).any(), (what, s, "unwritten or NaN")
        bad = got[i].view(np.uint32) != want.view(np.uint32)
        assert not bad.any(), (what, s, int(bad.sum()), np.argwhere(bad)[:3])


def nan_patterns(h, w):
    """(label, NaN mask) with NaN at the edges, in the corners and in whole rows."""
    m = np.zeros((h, w), bool)
    m[0, :] = m[:, -1] = True
    yield "edges", m
    m = np.zeros((h, w), bool)
    m[0, 0] = m[0, -1] = m[-1, 0] = m[-1, -1] = True
    m[:3, :3] = True
    yield "corners", m
    m = np.zeros((h, w), bool)
    m[h // 3] = m[h // 3 + 1] = m[-1] = True
    yield "rows", m


@pytest.mark.parametrize("n_sigma", [1, 2])
def test_gaussian_fills_nan_bit_for_bit(n_sigma):
    h, w = 37, 53
    base = field(701, h, w, 150.0, 400.0)
    sigmas = (6.0, 1.2) if n_sigma == 2 else (0.8,)
    for label, mask in nan_patterns(h, w):
        x = base.copy()
        x[mask] = np.nan
        median = K.nan_fill(x)
        assert median % 1 != 0                                # a fractional fill
        for fill in (-123.5, 0.0, median):
            assert_scipy_bits(run_gaussian(x, sigmas, fill), x, sigmas, fill, (label, fill))
    assert_scipy_bits(run_gaussian(base, sigmas), base, sigmas, None, "no NaN, replace_nan = 0")


@pytest.mark.parametrize("shape", [(1, 37), (41, 1), (2, 2), (5, 7), (64, 48)])
def test_gaussian_one_tap_and_radius_96(shape):
    """sigma 0 is one tap (scipy leaves the axis as it is); sigma 23.9 is radius 96, the largest the kernel takes, which on
    these images reflects around the edges several times."""
    x = field(shape[0] * 97 + shape[1], *shape, -20.0, 300.0)
    assert int(4 * 23.9 + 0.5) == 96
    for sigmas in ((0.0,), (23.9,), (0.0, 23.9), (23.9, 1e-16)):
        assert_scipy_bits(run_gaussian(x, sigmas), x, sigmas, None, (shape, sigmas))
    x[0, 0] = np.nan
    assert_scipy_bits(run_gaussian(x, (23.9, 0.0), -7.25), x, (23.9, 0.0), -7.25, (shape, "NaN"))


@pytest.mark.parametrize("n", [1024, 4096])
def test_gaussian_at_product_sizes(n):
    x = field(n, n, n, 100.0, 900.0)
    x[n // 2, :] = np.nan
    x[:, :5] = np.nan
    fill = K.nan_fill(x)
    assert_scipy_bits(run_gaussian(x, (6.0, 1.2), fill), x, (6.0, 1.2), fill, n)


def test_gaussian_argument_errors_return_before_any_launch():
    h, w = 8, 9
    xd = dev(field(5, h, w))
    tmp = Guarded((2, h, w), torch.float32, DEV)
    out = Guarded((2, h, w), torch.float32, DEV)
    good, good_r = taps_of((1.2, 6.0))
    asym = good.copy()
    asym[0] *= 1.0 + 1e-9
    wide = np.ones(2 * 97 + 1)
    cases = [
        ("asymmetric taps", dict(taps=(asym, good_r)), "not symmetric"),
        ("radius 97", dict(taps=(wide, [97]), n_sigma=1), "radius 97 outside"),
        ("n_sigma 0", dict(n_sigma=0), "n_sigma=0"),
        ("n_sigma 3", dict(n_sigma=3), "n_sigma=3"),
        ("x aliases tmp", dict(tmp=xd.data_ptr()), "aliased"),
        ("x aliases out", dict(out=xd.data_ptr()), "aliased"),
        ("tmp aliases out", dict(out=tmp.data_ptr()), "aliased"),
        ("h > 65535", dict(h=65536, w=1), "bad shape 65536 x 1"),
    ]
    for label, kw, message in cases:
        w64, radius = kw.get("taps", (good, good_r))
        rc = gaussian_call(xd.data_ptr(), kw.get("h", h), kw.get("w", w), 0, 0.0, kw.get("n_sigma", 2), w64, radius,
                           kw.get("tmp", tmp.data_ptr()), kw.get("out", out.data_ptr()))
        err = L.lib().tdx_last_error().decode()
        assert rc != 0 and message in err, (label, rc, err)
        torch.cuda.synchronize()
        for g in (tmp, out):
            g.check(label)
            assert torch.isnan(g.view).all(), f"{label}: a kernel ran"


# ---------------------------------------------------------------------------------------------------------------- shade

def with_nan(e, frac_seed, fill_sign):
    """e with ~6% of the pixels NaN; the NaN-median fill then has the sign of the field's median."""
    e = e.copy()
    rng = np.random.RandomState(frac_seed)
    e.flat[rng.choice(e.size, e.size // 16, replace=False)] = np.nan
    assert np.sign(K.nan_fill(e)) == fill_sign
    return e


def with_inf(e):
    e = e.copy()
    e[3, 4] = np.inf
    e[-5, -7] = -np.inf
    return e


def deep(h, w):
    return field(907, h, w, -5000.0, 4000.0)


# name: (elevation builder, get_relief_map keywords, what the case must reach: f(contract, shade args, elevation))
SHADE_CASES = {
    "stats_range_vmin_zero": (lambda: field(901, 64, 80, 300.0, 600.0), {},
                              lambda c, a, e: c["ocean"].any() and (~c["ocean"]).any() and K.decode_range(
                                  a["stats"], 0, 0, 0, 0)[2]),
    "stats_range_land": (lambda: field(902, 48, 64, 2000.0, 300.0), {},
                         lambda c, a, e: not K.decode_range(a["stats"], 0, 0, 0, 0)[2]),
    "user_range": (lambda: field(903, 48, 64, 500.0, 400.0), {"vmin": 300.0, "vmax": 1800.5},
                   lambda c, a, e: a["user_range"] and not a["vmin_is_zero"] and np.isnan(c["xa"]).any()),
    "user_range_vmin_zero": (lambda: field(904, 48, 64, 500.0, 400.0), {"vmin": -50.0, "vmax": 900.0},
                             lambda c, a, e: a["user_range"] and a["vmin_is_zero"]),
    "vmin_above_all_land": (lambda: field(905, 40, 56, 300.0, 500.0), {"vmin": 1e5, "vmax": 2e5},
                            lambda c, a, e: np.isnan(c["xa"][~c["ocean"]]).all() and
                            np.all(c["rgb"][~c["ocean"]] == 0)),
    "xa_256": (lambda: field(906, 40, 56, 900.0, 500.0), {"vmin": 0.0, "vmax": 700.0},
               lambda c, a, e: (c["xa"] == 256).any()),
    "flat": (lambda: np.full((40, 56), 850.0, F32), {}, lambda c, a, e: K.is_fallback(*K.decode_stats(a["stats"]))),
    "all_ocean": (lambda: field(908, 40, 48, -3000.0, 400.0), {},
                  lambda c, a, e: c["ocean"].all() and K.is_fallback(*K.decode_stats(a["stats"]))),
    "inf": (lambda: with_inf(field(909, 48, 64, 400.0, 300.0)), {"sigma_large": 1.5, "sigma_small": 0.5},
            lambda c, a, e: K.is_fallback(*K.decode_stats(a["stats"])) and np.isinf(e).sum() == 2),
    "all_nan": (lambda: np.full((12, 20), np.nan, F32), {},
                lambda c, a, e: a["replace_nan"] and np.isnan(c["rgb"]).all()),
    "nan_positive_fill": (lambda: with_nan(field(910, 48, 64, 400.0, 300.0), 1, 1), {},
                          lambda c, a, e: a["nan_fill"] > 0 and np.isnan(c["rgb"][np.isnan(e)]).all()),
    "nan_negative_fill": (lambda: with_nan(field(911, 48, 64, -400.0, 300.0), 2, -1), {},
                          lambda c, a, e: a["nan_fill"] < 0 and not np.isnan(c["rgb"]).any()),
    "below_minus_10000": (lambda: deep(48, 64), {}, lambda c, a, e: (e < -10000).any() and (e > 0).any()),
    "relief_0": (lambda: field(912, 48, 64, 200.0, 500.0), {"relief": 0.0}, lambda c, a, e: True),
    "relief_0.7_res30": (lambda: field(913, 48, 64, 200.0, 500.0), {"relief": 0.7, "resolution": 30},
                         lambda c, a, e: True),
    "relief_1.5": (lambda: field(914, 48, 64, 200.0, 500.0), {"relief": 1.5}, lambda c, a, e: True),
    # the gain is relief * (0.35 + 0.65 hill) + 1 - relief >= 1 - 0.65 relief: negative only above relief 1.54, above
    # 1 only for a negative relief
    "relief_2_gain_below_0": (lambda: field(915, 48, 64, 200.0, 900.0), {"relief": 2.0},
                              lambda c, a, e: (c["gain"] < 0).any() and (c["rgb"] == 0).any()),
    "relief_-0.5_gain_above_1": (lambda: field(916, 48, 64, 200.0, 500.0), {"relief": -0.5},
                                 lambda c, a, e: (c["gain"] > 1).any() and (c["rgb"] == 1).any()),
    "az45_res30": (lambda: field(917, 48, 64, 200.0, 500.0), {"azimuths": (45.0,), "resolution": 30},
                   lambda c, a, e: True),
    "az200_sigmas": (lambda: field(918, 48, 64, 200.0, 500.0),
                     {"azimuths": (200.0, 10.0), "sigma_large": 3.0, "sigma_small": 0.0}, lambda c, a, e: True),
    "h2": (lambda: field(919, 2, 37, 100.0, 400.0), {}, lambda c, a, e: True),
    "w2": (lambda: field(920, 41, 2, 100.0, 400.0), {}, lambda c, a, e: True),
    "2x2": (lambda: field(921, 2, 2, -10.0, 400.0), {}, lambda c, a, e: True),
    "1024^2": (lambda: field(922, 1024, 1024, 300.0, 800.0), {}, lambda c, a, e: True),
    "4096^2": (lambda: field(923, 4096, 4096, 300.0, 800.0), {}, lambda c, a, e: True),
}


def run_shade(args: dict, stats_dev) -> np.ndarray:
    """tdx_relief_shade with the contract's arguments into a guarded buffer pre-filled with UNWRITTEN."""
    e = args["elev"]
    h, w = e.shape
    ed, bd = dev(e), dev(args["blurred"])
    lut = dev(K.LUT32)
    out = Guarded((h, w, 3), torch.float32, DEV)
    out.view.fill_(UNWRITTEN)
    L.call(L.lib().tdx_relief_shade, DEV, ed.data_ptr(), bd.data_ptr(), stats_dev, lut.data_ptr(), h, w,
           args["replace_nan"], float(args["nan_fill"]), float(args["grad_div"]), args["az"], args["sin_alt"],
           args["cos_alt"], float(args["relief"]), float(args["one_minus_relief"]), args["user_range"],
           float(args["vmin"]), float(args["denom"]), args["vmin_is_zero"], out.data_ptr())
    got = fetch(out, "shade out")
    assert not (got == UNWRITTEN).any(), "unwritten pixels"
    return got


def check_against_contract_and_oracle(got, e, kw, contract, what):
    """Bit for bit against the contract except its excused pixels, and all pixels under the oracle rule; returns the
    line to report."""
    assert np.array_equal(np.isnan(got), np.isnan(contract["rgb"])), what
    bad = K.mismatches(got, contract)
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:4].tolist())
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        parts = O.relief_parts(e, **kw)
    n_boundary, share = K.compare(got, parts["rgb"], parts)
    d, (r, c), on_boundary = K.worst_pixel(got, parts["rgb"], parts)
    return (f"{what}: {K.excuse_summary(contract)}; vs oracle {n_boundary} LUT-boundary px, worst share of the "
            f"{K.TOL:g} bound {share:.3f}, worst |diff| {d:.3g} at ({r}, {c}) "
            f"{'on' if on_boundary else 'off'} a colormap boundary")


@pytest.mark.parametrize("name", list(SHADE_CASES))
def test_shade_is_the_contract(name, notes):
    build, kw, reaches = SHADE_CASES[name]
    e = build()
    args = K.shade_args(e, **kw)
    # the statistics from the device, which test_stats_counts_and_extrema_exactly pins to encode_stats
    stats = run_stats(e)
    assert np.array_equal(stats, args["stats"])
    stats_dev = torch.from_numpy(stats.view(np.int32).copy()).to(DEV)
    contract = K.shade(**args)
    assert reaches(contract, args, e), f"{name} does not reach its branch"
    got = run_shade(args, stats_dev.data_ptr())
    notes.append("shade " + check_against_contract_and_oracle(got, e, kw, contract, f"{name} {e.shape}"))
    if args["user_range"]:                                # the statistics are not read: a null pointer is accepted
        again = run_shade(args, 0)
        assert np.array_equal(again.view(np.uint32), got.view(np.uint32))


# ------------------------------------------------------------------------------------------------ the product sizes

@pytest.mark.parametrize("n", [512, 1024])
def test_benchmark_field_through_get_relief_map(n, notes):
    e = bench_field(n)
    got = get_relief_map(e, None, None, None)
    contract = K.relief_contract(e)
    notes.append("get_relief_map " + check_against_contract_and_oracle(got, e, {}, contract, f"benchmark field {n}^2"))
