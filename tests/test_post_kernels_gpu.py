"""The seven elevation / climate read-out kernels of csrc/tdx_post.cu, each through its C entry point, compared two ways:

(a) bit for bit with an fp32 restatement that rounds once per operation in the kernel's order (oracle/postproc.py where
    it already is that restatement, otherwise restated here).  Bit patterns are compared, so -0.0 vs +0.0 is a
    difference and NaN must appear in exactly the restatement's positions;
(b) against a plain fp64 evaluation of the same mathematics, within a per-element bound gamma_n * sum|terms| (Higham's
    gamma_n = n u / (1 - n u), u = 2^-24, n = the rounded operations on the longest path, derived beside each bound).

(b) catches an error the kernel shares with the oracle; (a) catches an operand swap or a wrong edge index that stays
inside a loose bound.  Every output lives in a guarded, NaN-filled buffer (tests/_igemm_ref.Guarded): a write outside
the tensor, or an element left unwritten, fails.  The worst share of each bound is written to the terminal."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import postproc as P
from terrain_diffusion_b200 import _lib as L
from tests._igemm_ref import Guarded, report
from tests._post_inputs import coastal_coarse_map, field

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
U = 2.0 ** -24


def gamma(n: int) -> float:
    return n * U / (1.0 - n * U)


@pytest.fixture(scope="module")
def margins(request):
    """Worst measured share of each fp64 bound below; written to the terminal (also under -q) when the module is done."""
    found: dict = {}
    yield found
    report(request.config, [f"worst {kind}: {v:.3g} of the bound" for kind, v in sorted(found.items())])


def dev(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).to(DEV)


def out_buf(shape) -> Guarded:
    return Guarded(tuple(shape), torch.float32, DEV)


class Guarded16:
    """Guarded for int16: 0x2A2A sentinels on both sides, the view filled with 0x7EAD (a value no case here packs)."""

    def __init__(self, shape):
        self.numel, self.pad = int(np.prod(shape)), 64
        self.raw = torch.full((2 * self.pad + self.numel,), 0x2A2A, dtype=torch.int16, device=DEV)
        self.view = self.raw[self.pad:self.pad + self.numel].view(*shape)
        self.view.fill_(0x7EAD)

    def data_ptr(self):
        return self.view.data_ptr()

    def check(self, what):
        guards = torch.cat([self.raw[:self.pad], self.raw[self.pad + self.numel:]])
        assert bool((guards == 0x2A2A).all()), f"{what}: written outside the tensor"
        assert not bool((self.view == 0x7EAD).any()), f"{what}: an element was not written"


def launch(fn, *args):
    L.call(fn, DEV, *args)
    torch.cuda.synchronize()


def fetch(g: Guarded, what: str) -> np.ndarray:
    torch.cuda.synchronize()
    g.check(what)
    return g.view.cpu().numpy()


def assert_bits(got: np.ndarray, want: np.ndarray, what: str):
    """Bit-identical wherever `want` is not NaN; NaN in exactly the same positions."""
    want = np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_g, nan_w), f"{what}: NaN positions differ at {int((nan_g ^ nan_w).sum())} elements"
    diff = (got.view(np.uint32) != want.view(np.uint32)) & ~nan_w
    if diff.any():
        i = tuple(int(v) for v in np.argwhere(diff)[0])
        raise AssertionError(f"{what}: {int(diff.sum())} of {int((~nan_w).sum())} elements differ in their bits; first at "
                             f"{i}: got {got[i]!r}, want {want[i]!r}")


def assert_within(got: np.ndarray, ref: np.ndarray, bound: np.ndarray, what: str, margins: dict, kind: str):
    """|got - ref| <= bound element by element (ref in fp64); a non-finite ref must be matched exactly (NaN by
    position, +-inf by value).  Records the worst err / bound under `kind`."""
    got, ref = got.astype(np.float64), np.asarray(ref, np.float64)
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}: NaN positions differ from the fp64 evaluation"
    assert np.array_equal(got[~fin & ~np.isnan(ref)], ref[~fin & ~np.isnan(ref)]), f"{what}: infinities differ"
    err, b = np.abs(got[fin] - ref[fin]), np.asarray(np.broadcast_to(bound, ref.shape))[fin]
    assert np.isfinite(got[fin]).all(), f"{what}: non-finite result where the fp64 value is finite"
    bad = err > b
    if bad.any():
        k = int(np.argmax(np.where(b > 0, err / np.where(b > 0, b, 1), np.inf)))
        raise AssertionError(f"{what}: {int(bad.sum())} elements outside the fp64 bound; worst err {err[k]:.3g} "
                             f"vs bound {b[k]:.3g}")
    share = float((err / np.where(b > 0, b, 1.0)).max()) if err.size else 0.0
    margins[kind] = max(margins.get(kind, 0.0), share)


# ------------------------------------------------------------------------------------------------ post_normalize
@pytest.mark.parametrize("w", [1, 127, 128, 129, 300])
@pytest.mark.parametrize("extra", [0, 13])
@pytest.mark.parametrize("scale,offset", [(1.35, 0.12), (-38.6, -31.4)])
def test_post_normalize(w, extra, scale, offset, margins):
    h, pitch = 5, w + extra
    num = np.full((h, pitch), np.nan, F32)                  # the pitch padding is NaN: reading it would show
    den = np.full((h, pitch), np.nan, F32)
    num[:, :w] = field(11, h, w, 0.0, 3.0)
    den[:, :w] = 0.5 + np.abs(field(12, h, w))
    den[0, :w:3] = 0.0                                      # x / 0 -> +-inf
    den[1, :w:2], num[1, :w:2] = 0.0, 0.0                   # 0 / 0 -> NaN
    num[2, :w:4] = -0.0                                     # -0 / d -> -0
    den[3, :w:2] *= -1.0
    out = out_buf((h, w))
    nd, dd = dev(num), dev(den)
    launch(L.lib().tdx_post_normalize, nd.data_ptr(), dd.data_ptr(), pitch, out.data_ptr(), h, w, scale, offset)
    got = fetch(out, "post_normalize")
    n, d, s, o = num[:, :w], den[:, :w], F32(scale), F32(offset)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = (n / d).astype(F32)
        assert_bits(got, ((q * s).astype(F32) + o).astype(F32), f"post_normalize w={w} pitch={pitch}")
        q64 = n.astype(np.float64) / d.astype(np.float64)
        ref = q64 * float(s) + float(o)
    # three roundings (divide, multiply, add) on one path: gamma_3 * (|n/d * scale| + |offset|)
    bound = gamma(3) * (np.abs(q64 * float(s)) + abs(float(o)))
    assert_within(got, ref, bound, f"post_normalize w={w} pitch={pitch}", margins, "post_normalize")


# ------------------------------------------------------------------------------------------------ post_pad_extrapolate
def _pad64(x: np.ndarray, sign: float) -> np.ndarray:
    """pad_linear_extrapolation in fp64; sign = +1 turns every difference into a sum, which on |x| gives sum|terms|."""
    h, w = x.shape
    top = 2 * x[0:1] + sign * x[1:2] if h > 1 else x[0:1]
    bot = 2 * x[-1:] + sign * x[-2:-1] if h > 1 else x[-1:]
    x = np.concatenate([top, x, bot], axis=0)
    left = 2 * x[:, 0:1] + sign * x[:, 1:2] if w > 1 else x[:, 0:1]
    right = 2 * x[:, -1:] + sign * x[:, -2:-1] if w > 1 else x[:, -1:]
    return np.concatenate([left, x, right], axis=1)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 5), (5, 1), (2, 2), (2, 131), (131, 2), (37, 53)])
def test_post_pad_extrapolate(h, w, margins):
    x = field(21 + h, h, w, -3.0, 40.0)
    out = out_buf((h + 2, w + 2))
    xd = dev(x)
    launch(L.lib().tdx_post_pad_extrapolate, xd.data_ptr(), h, w, out.data_ptr())
    got = fetch(out, "pad")
    assert_bits(got, P.pad_linear_extrapolation(x), f"pad {h}x{w}")
    # an edge is one rounded subtraction (2x is exact), a corner extrapolates two of those: gamma_2 * sum|terms|
    x64 = x.astype(np.float64)
    assert_within(got, _pad64(x64, -1.0), gamma(2) * _pad64(np.abs(x64), 1.0), f"pad {h}x{w}", margins,
                  "post_pad_extrapolate")


# ------------------------------------------------------------------------------------------------ resize_aa_axis
def _resize64(x: np.ndarray, out_size: int, axis: int):
    """The triangle filter with exact weights (fp64) along `axis`, and the bound on the kernel's error.

    The kernel's weight for tap J is 1 - |fl(fl(fl(J - center_f) + 0.5) * invscale_f)| with center_f = fl(fl(in/out) *
    (i + 0.5)) (2 roundings from the exact center c) and invscale_f = fl(1 / fl(in/out)) (2 roundings from 1/scale).
    Summing the rounding of each step scaled to t gives |t_f - t| <= gamma_7 * invscale * (J + c + 1), and the final
    1 - t adds one more: delta_J = gamma_8 * (invscale * (J + c + 1) + 1) bounds each weight's absolute error (a tap the
    fp32 support test drops has exact weight below delta_J).  Normalising by the fp32 total (n - 1 additions off by at
    most D = sum delta + gamma_n * total) and one division give the normalised weight error
    dW_J = (delta_J + W_J D) / (total - D) + u (W_J + ...), and the n products and n - 1 additions of the tap sum add
    gamma_{n+1} * sum |x_J| W_J."""
    in_size = x.shape[axis]
    scale = in_size / out_size
    support = max(scale, 1.0)
    inv = 1.0 / scale if scale >= 1.0 else 1.0
    i = np.arange(out_size, dtype=np.float64)[:, None]
    J = np.arange(in_size, dtype=np.float64)[None, :]
    c = scale * (i + 0.5)
    wgt = np.maximum(0.0, 1.0 - np.abs(J - c + 0.5) * inv)
    total = wgt.sum(axis=1, keepdims=True)
    W = wgt / total
    n = int(np.ceil(support)) * 2 + 1
    delta = gamma(8) * (inv * (J + c + 1.0) + 1.0) * (np.abs(J + 0.5 - c) * inv <= 1.0 + 1e-3)
    D = delta.sum(axis=1, keepdims=True) + gamma(n) * total
    dW = (delta + W * D) / (total - D)
    dW = dW + gamma(1) * (W + dW)
    xm = np.moveaxis(x.astype(np.float64), axis, -1)
    ref = xm @ W.T
    bound = np.abs(xm) @ (dW + gamma(n + 1) * (W + dW)).T
    return np.moveaxis(ref, -1, axis), np.moveaxis(bound, -1, axis)


def _signed_zero_runs(x: np.ndarray, axis: int) -> np.ndarray:
    """Runs of -0.0 and +0.0 along the resized axis, and one whole line of -0.0 across it."""
    x = np.moveaxis(x.copy(), axis, -1)
    n = x.shape[-1]
    x[..., n // 4:n // 2] = -0.0
    x[..., (3 * n) // 4:] = 0.0
    x[0] = -0.0
    return np.moveaxis(x, -1, axis)


def _check_resize(x, out_size, axis, margins, what):
    h, w = x.shape
    oshape = (out_size, w) if axis == 0 else (h, out_size)
    out = out_buf(oshape)
    xd = dev(x)
    launch(L.lib().tdx_resize_aa_axis, xd.data_ptr(), h, w, out.data_ptr(), out_size, axis)
    got = fetch(out, what)
    assert_bits(got, P._resize_axis(x, out_size, axis), what)
    ref, bound = _resize64(x, out_size, axis)
    assert_within(got, ref, bound, what, margins, "resize_aa_axis")


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("in_size", range(1, 25))
def test_resize_every_small_pair(in_size, axis, margins):
    for out_size in range(1, 25):
        shape = (in_size, 3) if axis == 0 else (3, in_size)
        x = field(31 + in_size, *shape, 0.5, 2.0)
        _check_resize(x, out_size, axis, margins, f"resize axis {axis} {in_size}->{out_size}")
        if in_size >= 4:
            _check_resize(_signed_zero_runs(x, axis), out_size, axis, margins,
                          f"resize axis {axis} {in_size}->{out_size} signed zeros")


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("in_size,out_size", [(512, 7), (7, 512), (96, 80), (80, 96), (17, 130), (64, 1), (1, 64),
                                              (23, 17), (13, 200), (8, 64)])
def test_resize_large_and_coprime(in_size, out_size, axis, margins):
    shape = (in_size, 131) if axis == 0 else (9, in_size)     # 131 / 130 wide: a second block column
    x = field(41 + in_size, *shape, -20.0, 30.0)
    _check_resize(x, out_size, axis, margins, f"resize axis {axis} {in_size}->{out_size}")
    _check_resize(_signed_zero_runs(x, axis), out_size, axis, margins,
                  f"resize axis {axis} {in_size}->{out_size} signed zeros")


# ------------------------------------------------------------------------------------------------ gaussian_blur
def _blur(x: np.ndarray, ksize: int, sigma: float) -> np.ndarray:
    out = out_buf(x.shape)
    xd = dev(x)
    launch(L.lib().tdx_gaussian_blur, xd.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(), ksize, sigma)
    return fetch(out, f"blur k={ksize}")


def _blur_fp32(x: np.ndarray, K: np.ndarray) -> np.ndarray:
    """The kernel's order: reflect padding, taps row-major, acc = fl(acc + fl(K[dy, dx] * x)) from +0."""
    k = K.shape[0]
    p = k // 2
    xp = np.pad(x.astype(F32), p, mode="reflect")
    h, w = x.shape
    acc = np.zeros((h, w), F32)
    for dy in range(k):
        for dx in range(k):
            acc = (acc + (K[dy, dx] * xp[dy:dy + h, dx:dx + w]).astype(F32)).astype(F32)
    return acc


def _taps64(ksize: int, sigma: float):
    """The fp64 Gaussian taps (on the fp32 sigma the kernel receives) and each tap's relative error bound.

    The host computes t = fl((i - half) / sigma), z = -0.5 * fl(t * t) (3 roundings relative to z: |dz| <= 3u|z|),
    expf(z) (glibc: under 1 ulp, <= 2u), the sequential fp32 sum S of k taps (gamma_{k-1}, plus the taps' own errors
    weighted by the taps: A) and one division.  So tap i is off by at most r_i = (3|z_i| + 2) u + (k - 1) u + A + u
    relative to its exact value, and fl(k_i k_j) by r_i + r_j + u; expf results below the normal range add an absolute
    error under 2^-148."""
    s = float(F32(sigma))
    half = (ksize - 1) * 0.5
    z = -0.5 * ((np.arange(ksize) - half) / s) ** 2
    e = np.exp(z)
    k = e / e.sum()
    own = (3.0 * np.abs(z) + 2.0) * U
    A = float((e * own).sum() / e.sum())
    r = own + (ksize - 1) * U + A + U
    return k, r


@pytest.mark.parametrize("sigma", [0.8, 5.0, 7.3])
@pytest.mark.parametrize("ksize", [1, 3, 11, 31])
def test_gaussian_blur(ksize, sigma, margins):
    p = ksize // 2
    # the 2-D table the kernel uses, read off its response to a unit impulse: every other term adds K * 0 = +0
    side = 2 * ksize + 1
    imp = np.zeros((side, side), F32)
    imp[ksize, ksize] = 1.0
    resp = _blur(imp, ksize, sigma)
    K = resp[ksize + p - np.arange(ksize)[:, None], ksize + p - np.arange(ksize)[None, :]]
    assert np.isfinite(K).all() and (K >= 0).all()
    assert_bits(resp, _blur_fp32(imp, K), f"blur impulse k={ksize} sigma={sigma}")
    k64, r = _taps64(ksize, sigma)
    K64 = np.outer(k64, k64)
    tbound = K64 * (r[:, None] + r[None, :] + U) * (1 + 1e-6) + 2.0 ** -148
    assert_within(K, K64, tbound, f"blur taps k={ksize} sigma={sigma}", margins, "gaussian_blur taps")

    shapes = [(p + 1, 40), (40, p + 1), (40, 300), (17, 36)]
    for h, w in shapes:
        x = field(51 + h + w, h, w, -30.0, 40.0)
        got = _blur(x, ksize, sigma)
        what = f"blur k={ksize} sigma={sigma} {h}x{w}"
        assert_bits(got, _blur_fp32(x, K), what)
        # fp64: sum K64 * x over the reflected window.  Each table entry is off by tbound, then one product and k^2
        # additions: gamma_{k^2+1} on every term
        xp = np.pad(x.astype(np.float64), p, mode="reflect")
        ref, bound = np.zeros((h, w)), np.zeros((h, w))
        for dy in range(ksize):
            for dx in range(ksize):
                v = xp[dy:dy + h, dx:dx + w]
                ref += K64[dy, dx] * v
                bound += np.abs(v) * (tbound[dy, dx] + gamma(ksize * ksize + 1) * (K64[dy, dx] + tbound[dy, dx]))
        assert_within(got, ref, bound, what, margins, "gaussian_blur")
    if p:
        out = out_buf((p, 40))
        xd = dev(np.zeros((p, 40), F32))
        rc = L.lib().tdx_gaussian_blur(xd.data_ptr(), p, 40, out.data_ptr(), ksize, sigma, L.current_stream_ptr())
        assert rc != 0 and b"reflect" in L.lib().tdx_last_error()


# ------------------------------------------------------------------------------------------------ post_combine
EDGES = [0.0, -0.0, np.nan, np.inf, -np.inf, -32768.5, -32769.0, 32767.9, 32768.0, -32768.0, 2.0 ** 23, 2.0 ** 23 + 1,
         -(2.0 ** 24), 3.0e9, -1e-30, -1e-45, -1e-20, 181.02, -181.02, 181.0, -181.0, 1.5, -1.5, -0.5]


@pytest.mark.parametrize("signed_square", [0, 1])
@pytest.mark.parametrize("outputs", ["float", "int16", "both"])
def test_post_combine(signed_square, outputs, margins):
    h, w, ap, bp = 4, 133, 140, 150
    a = np.full((h, ap), np.nan, F32)
    b = np.full((h, bp), np.nan, F32)
    a[:, :w] = field(61, h, w, 0.0, 200.0)
    b[:, :w] = field(62, h, w, 0.0, 50.0)
    ne = len(EDGES)
    a[0, :ne], b[0, :ne] = EDGES, 0.0                      # the edge values as they are (b = +0)
    a[1, :ne], b[1, :ne] = EDGES, -0.0                     # ... plus -0: -0 + -0 stays -0
    a[2, :ne] = np.array(EDGES, F32) - b[2, :ne]           # ... as the rounded sum of two terms
    a[3, :4], b[3, :4] = [1e30, -1e30, 2.0 ** 24, -0.0], [1e30, 1e30, 1.0, 0.0]
    out = out_buf((h, w)) if outputs != "int16" else None
    o16 = Guarded16((h, w)) if outputs != "float" else None
    ad, bd = dev(a), dev(b)
    launch(L.lib().tdx_post_combine, ad.data_ptr(), ap, bd.data_ptr(), bp, out.data_ptr() if out else None,
           o16.data_ptr() if o16 else None, h, w, signed_square)
    aw, bw = a[:, :w], b[:, :w]
    with np.errstate(over="ignore", invalid="ignore"):
        v = (aw + bw).astype(F32)
        want = (np.sign(v) * np.square(v)).astype(F32) if signed_square else v      # world_pipeline.py:1312
        s64 = aw.astype(np.float64) + bw.astype(np.float64)
        ref = np.sign(s64) * s64 * s64 if signed_square else s64
        ref = np.where(np.isinf(ref.astype(F32)), ref.astype(F32), ref)      # past the fp32 range: +-inf
    terms = np.abs(aw.astype(np.float64)) + np.abs(bw.astype(np.float64))
    # the add is one rounding (gamma_1 (|a| + |b|)); squaring the rounded sum adds one more on a squared value:
    # gamma_3 (|a| + |b|)^2
    # (+ 2^-149: a square that lands below the normal range is off by up to half a subnormal step)
    bound = gamma(3) * terms * terms + 2.0 ** -149 if signed_square else gamma(1) * terms
    what = f"post_combine signed_square={signed_square} {outputs}"
    if out is not None:
        got = fetch(out, what)
        assert_bits(got, want, what)
        with np.errstate(over="ignore", invalid="ignore"):
            assert_within(got, ref, bound, what, margins, "post_combine")
    if o16 is not None:
        g16 = fetch(o16, what + " int16")
        with np.errstate(invalid="ignore"):
            assert np.array_equal(g16, P.elev_to_int16(want)), what
        if not signed_square:
            assert g16[0, EDGES.index(-32768.5)] == -32768 and g16[0, EDGES.index(32767.9)] == 32767
            assert g16[0, 2] == 0 and g16[0, 3] == 32767 and g16[0, 4] == -32768    # NaN packs as 0, +-inf clip
            assert g16[0, EDGES.index(-1e-30)] == -1


# ------------------------------------------------------------------------------------------------ lapse_rate
BETA_LO, BETA_HI, FALLBACK, EPS = -0.012, 0.0, -0.0065, 1e-6


def _lapse_inputs(name):
    """(temperature, signed-sqrt coarse elevation, win, fallback_threshold)."""
    if name == "coastal":
        T, c0 = coastal_coarse_map()
        return T, c0, 15, 0.02
    rng = np.random.RandomState(len(name))
    h, w = (20, 160) if "wide" in name else (12, 14)
    c0 = field(71, h, w, 6.0, 14.0)
    T = field(72, h, w, 15.0, 5.0) - 0.006 * np.maximum(c0, 0) ** 2
    if "ocean" in name:                                    # no land at all: den = 0 in every window
        c0 = -(0.1 + np.abs(c0))
    else:                                                  # ocean patches: sparse-land windows on both sides of thr
        c0[rng.rand(h, w) < 0.55] *= -1.0
        c0[:, :3] = np.where(np.arange(h)[:, None] % 3 == 0, 1.0, -1.0)            # flat land next to ocean
        T[:4] = 10.0 + 0.05 * np.maximum(c0[:4], 0) ** 2                           # slope > 0: clipped at 0
    win = 3 if "win3" in name else 15
    return T.astype(F32), c0.astype(F32), win, 0.3 if win == 3 else 0.02


def _lapse64(T, c0, win, thr):
    """local_baseline_temperature in fp64 on the exact e = max(c0, 0)^2, with the kernel's error bound.

    Each window sum adds N = win^2 terms, each at most two roundings from its exact value (e = fl(c^2), e*e, e*T):
    gamma_{N+1}.  den = fl(count / N) and dd = fl(den + eps), and each mean divides twice: gamma_{N+5} * sum|terms| /
    N / (den + eps) per mean (E_X).  var and cov each add a product and a subtraction (gamma_2 on their terms) to the
    propagated mean errors, beta = cov / (var + eps) one more division, and T_sea = T - beta * e two more roundings."""
    T64, c = T.astype(np.float64), c0.astype(np.float64)
    e = np.where(c > 0, c * c, 0.0)
    m = (e > 0).astype(np.float64)
    N = win * win

    def pool(x):
        h, w = x.shape
        oh, ow = h - win + 1, w - win + 1
        return sum(x[dy:dy + oh, dx:dx + ow] for dy in range(win) for dx in range(win))

    den = pool(m) / N
    dd = den + float(F32(EPS))
    g = gamma(N + 5)
    mean = {k: pool(v * m) / N / dd for k, v in (("T", T64), ("e", e), ("e2", e * e), ("eT", e * T64))}
    err = {k: g * pool(np.abs(v) * m) / N / dd for k, v in (("T", T64), ("e", e), ("e2", e * e), ("eT", e * T64))}
    var = mean["e2"] - mean["e"] ** 2
    cov = mean["eT"] - mean["e"] * mean["T"]
    E_var = err["e2"] + (2 * np.abs(mean["e"]) + err["e"]) * err["e"] + gamma(2) * (np.abs(mean["e2"]) + mean["e"] ** 2)
    E_cov = (err["eT"] + np.abs(mean["e"]) * err["T"] + np.abs(mean["T"]) * err["e"] + err["e"] * err["T"]
             + gamma(2) * (np.abs(mean["eT"]) + np.abs(mean["e"] * mean["T"])))
    vd = var + float(F32(EPS))
    beta = cov / vd
    with np.errstate(divide="ignore", invalid="ignore"):
        E_beta = np.where(np.abs(vd) > E_var, (E_cov + np.abs(beta) * E_var) / (np.abs(vd) - E_var), np.inf)
    E_beta = E_beta + gamma(1) * np.abs(beta)
    invalid = (var < 1.0) | (den < float(F32(thr)))
    ambiguous = np.abs(var - 1.0) <= E_var
    beta = np.clip(np.where(invalid, float(F32(FALLBACK)), beta), float(F32(BETA_LO)), float(F32(BETA_HI)))
    p = (win - 1) // 2
    Tc, ec = T64[p:-p, p:-p], e[p:-p, p:-p]
    t_sea = Tc - beta * ec
    return beta, E_beta, invalid, ambiguous, t_sea, Tc, ec


@pytest.mark.parametrize("name", ["coastal", "win3", "win3_wide", "win15_wide", "win3_ocean", "win15_ocean_wide"])
def test_lapse_rate(name, margins):
    T, c0, win, thr = _lapse_inputs(name)
    h, w = T.shape
    oh, ow = h - win + 1, w - win + 1
    ts, be = out_buf((oh, ow)), out_buf((oh, ow))
    Td, cd = dev(T), dev(c0)
    launch(L.lib().tdx_lapse_rate, Td.data_ptr(), cd.data_ptr(), h, w, win, BETA_LO, BETA_HI, FALLBACK, EPS, thr,
           ts.data_ptr(), be.data_ptr())
    got_t, got_b = fetch(ts, f"lapse {name} t_sea"), fetch(be, f"lapse {name} beta")
    e = (np.sign(c0) * np.square(np.maximum(F32(0), c0))).astype(F32)           # world_pipeline.py:1329
    want_t, want_b = P.local_baseline_temperature(T, e, win, (BETA_LO, BETA_HI), FALLBACK, EPS, thr)
    assert_bits(got_b, want_b, f"lapse {name} beta")
    assert_bits(got_t, want_t, f"lapse {name} t_sea")

    beta64, E_beta, invalid64, ambiguous, t64, Tc, ec = _lapse64(T, c0, win, thr)
    fb = got_b == F32(FALLBACK)
    agree = (invalid64 == fb) | ambiguous                  # the fp32 and fp64 fallback decisions differ only where
    assert agree.all(), f"lapse {name}: fallback decisions differ"   # var_e is within its error bound of 1
    same = invalid64 == fb
    if "ocean" in name:
        assert fb.all()
    assert_within(got_b[same], beta64[same], np.where(invalid64, 0.0, E_beta)[same], f"lapse {name} beta", margins,
                  "lapse_rate beta")
    with np.errstate(invalid="ignore"):
        bound_t = np.where(invalid64 | (ec == 0), 0.0, ec * E_beta) + gamma(3) * (np.abs(Tc) + np.abs(beta64 * ec))
    assert_within(got_t[same], t64[same], bound_t[same], f"lapse {name} t_sea", margins, "lapse_rate t_sea")


# ------------------------------------------------------------------------------------------------ climate_sample
def _climate_case(name):
    """(i1, j1, h, w, S, ci1, cj1, hs, ws, crop, n_ch).  Unless a case shifts it, the geometry is compute_climate's:
    ci1 = i1 // S, hs = ceil(i2 / S) - ci1 + 2."""
    base = {"s256": (-37, 20, 128, 128, 256, 0, 0, 7, 6), "s64_wide": (-150, -200, 320, 430, 64, 0, 0, 7, 6),
            "one_cell": (5, 9, 20, 30, 64, 0, 0, 7, 6), "far_negative": (-70000, -70313, 40, 150, 256, 0, 0, 7, 6),
            "clamp_top_left": (10, 20, 50, 60, 64, 2, 2, 3, 7), "clamp_bottom_right": (10, 20, 50, 60, 64, -3, -3, 0, 6),
            "non_square": (-100, 300, 90, 140, 32, 0, 0, 5, 8)}[name]
    i1, j1, h, w, S, di, dj, crop, n_ch = base
    ci1, cj1 = i1 // S + di, j1 // S + dj
    hs, ws = -((-(i1 + h)) // S) - i1 // S + 2, -((-(j1 + w)) // S) - j1 // S + 2
    if name == "one_cell":
        hs = ws = 1
    if name == "clamp_bottom_right":
        hs, ws = 2, 3
    return i1, j1, h, w, S, ci1, cj1, hs, ws, crop, n_ch


def _bilinear64(f, sy, sx):
    """Bilinear sample of f [hs, ws] (fp64) at clamped coordinates; also sum |f| w and the local slopes."""
    hs, ws = f.shape
    y0, x0 = np.floor(sy).astype(int), np.floor(sx).astype(int)
    wy1, wx1 = sy - y0, sx - x0
    y1, x1 = np.minimum(y0 + 1, hs - 1), np.minimum(x0 + 1, ws - 1)
    val = ((1 - wy1) * (1 - wx1) * f[y0, x0] + (1 - wy1) * wx1 * f[y0, x1] + wy1 * (1 - wx1) * f[y1, x0]
           + wy1 * wx1 * f[y1, x1])
    a = np.abs(f)
    mag = (1 - wy1) * (1 - wx1) * a[y0, x0] + (1 - wy1) * wx1 * a[y0, x1] + wy1 * (1 - wx1) * a[y1, x0] + wy1 * wx1 * a[y1, x1]
    dy = np.zeros_like(f) if hs == 1 else np.abs(np.diff(f, axis=0))
    dx = np.zeros_like(f) if ws == 1 else np.abs(np.diff(f, axis=1))
    ly, lx = np.zeros(sy.shape), np.zeros(sx.shape)
    for oy in (-1, 0, 1):                                  # the slopes of every cell a perturbed point can fall in
        for ox in (-1, 0, 1, 2):
            r, q = np.clip(y0 + oy, 0, max(hs - 2, 0)), np.clip(x0 + ox, 0, ws - 1)
            if hs > 1:
                ly = np.maximum(ly, dy[r, q])
            r, q = np.clip(y0 + oy, 0, hs - 1), np.clip(x0 + ox, 0, max(ws - 2, 0))
            if ws > 1:
                lx = np.maximum(lx, dx[r, q])
    return val, mag, ly, lx


@pytest.mark.parametrize("name", ["s256", "s64_wide", "one_cell", "far_negative", "clamp_top_left",
                                  "clamp_bottom_right", "non_square"])
def test_climate_sample(name, margins):
    i1, j1, h, w, S, ci1, cj1, hs, ws, crop, n_ch = _climate_case(name)
    hc, wc = hs + 2 * crop, ws + 2 * crop
    t_sea = field(81, hs, ws, 14.0, 6.0)
    beta = (-0.012 * np.abs(field(82, hs, ws))).astype(F32)
    coarse = np.stack([field(90 + k, hc, wc, 0.0, 1.0 + k) for k in range(n_ch)]).astype(F32)
    elev = field(83, h, w, 200.0, 600.0)
    elev[0, :6] = [np.nan, -0.0, 0.0, np.inf, -np.inf, -5.0]
    out = out_buf((5, h, w))
    bufs = [dev(a) for a in (t_sea, beta, coarse, elev)]
    launch(L.lib().tdx_climate_sample, bufs[0].data_ptr(), bufs[1].data_ptr(), bufs[2].data_ptr(), n_ch, hc, wc, crop,
           bufs[3].data_ptr(), i1, j1, h, w, S, ci1, cj1, out.data_ptr())
    got = fetch(out, f"climate {name}")

    # (a) the restatement of compute_climate's sampling (oracle/postproc.py) on these planes
    ii = np.arange(i1, i1 + h, dtype=np.int64)[:, None] + np.zeros((1, w), np.int64)
    jj = np.arange(j1, j1 + w, dtype=np.int64)[None, :] + np.zeros((h, 1), np.int64)
    u = (((ii.astype(F32) + F32(0.5)) / F32(S)) - F32(ci1) + F32(0.5)).astype(F32)
    v = (((jj.astype(F32) + F32(0.5)) / F32(S)) - F32(cj1) + F32(0.5)).astype(F32)
    gy = (((u + F32(0.5)) * F32(2.0)) / F32(hs) - F32(1.0)).astype(F32)
    gx = (((v + F32(0.5)) * F32(2.0)) / F32(ws) - F32(1.0)).astype(F32)
    central = coarse[:, crop:crop + hs, crop:crop + ws]
    up = P._grid_sample_border(np.concatenate([t_sea[None], beta[None], central]).astype(F32), gy, gx)
    with np.errstate(invalid="ignore"):
        t_real = (up[0] + up[1] * np.maximum(elev, F32(0.0))).astype(F32)
    want = np.stack([t_real, up[5], up[6], up[7], up[1]])
    assert_bits(got, want, f"climate {name}")
    if name.startswith("clamp"):                           # every sample point really is clamped
        sy = ((gy + 1) * hs - 1) / 2
        sx = ((gx + 1) * ws - 1) / 2
        assert ((sy < 0) if "top" in name else (sy > hs - 1)).all()
        assert ((sx < 0) if "left" in name else (sx > ws - 1)).all()

    # (b) fp64: the exact sample point is u itself (unnormalize(gy) = u), clamped to [0, hs - 1].  The 11 rounded steps
    # from the pixel index to fp32 sy each err by u times an intermediate no larger than |i + 0.5| / S, |ci1|,
    # |u| + 1 or hs / 2 (in sy units), so |sy_f - sy| <= gamma_11 * (2 A + |ci1| + 6 (|u| + 1) + hs) = Dy; the result
    # moves by at most Dy times the largest step between neighbouring samples, plus the bilinear evaluation: one
    # rounding in 1 - w, one per weight product, one per tap product and three additions, gamma_6 * sum |f| w.
    u64 = (ii + 0.5) / S - ci1 + 0.5
    v64 = (jj + 0.5) / S - cj1 + 0.5
    sy64, sx64 = np.clip(u64, 0, hs - 1), np.clip(v64, 0, ws - 1)
    Dy = gamma(11) * (2 * np.abs(ii + 0.5) / S + abs(ci1) + 6 * (np.abs(u64) + 1) + hs)
    Dx = gamma(11) * (2 * np.abs(jj + 0.5) / S + abs(cj1) + 6 * (np.abs(v64) + 1) + ws)
    planes = [t_sea, beta, central[3], central[4], central[5]]
    res = [_bilinear64(f.astype(np.float64), sy64, sx64) for f in planes]
    E = [Dy * ly + Dx * lx + gamma(6) * mag for _, mag, ly, lx in res]
    e64 = elev.astype(np.float64)
    with np.errstate(invalid="ignore"):
        ep = np.where(np.isnan(e64), np.nan, np.maximum(e64, 0.0))
        t64 = res[0][0] + res[1][0] * ep
        # two more roundings (product, sum) on top of the sampled values' errors
        Et = E[0] + E[1] * np.abs(ep) + gamma(2) * (np.abs(res[0][0]) + np.abs(res[1][0] * ep))
    for k, (ref, bound) in enumerate([(t64, Et), (res[2][0], E[2]), (res[3][0], E[3]), (res[4][0], E[4]),
                                      (res[1][0], E[1])]):
        fin = np.isfinite(bound)
        with np.errstate(invalid="ignore"):
            assert_within(got[k][fin], ref[fin], bound[fin], f"climate {name} channel {k}", margins, "climate_sample")


# ------------------------------------------------------------------------------------------------ argument checks
def test_entry_points_reject_bad_shapes_before_launching():
    """Every entry point returns non-zero with a message, and writes nothing, for each shape it cannot run."""
    lib = L.lib()
    src = dev(np.ones(4096, F32))
    out = out_buf((4096,))
    x, o = src.data_ptr(), out.data_ptr()
    s = L.current_stream_ptr()
    bad = {
        "post_normalize h > 65535": lambda: lib.tdx_post_normalize(x, x, 8, o, 65536, 8, 1.0, 0.0, s),
        "post_normalize pitch < w": lambda: lib.tdx_post_normalize(x, x, 7, o, 4, 8, 1.0, 0.0, s),
        "pad h + 2 > 65535": lambda: lib.tdx_post_pad_extrapolate(x, 65534, 1, o, s),
        "resize > 65535 rows": lambda: lib.tdx_resize_aa_axis(x, 4, 4, o, 65536, 0, s),
        "resize axis 2": lambda: lib.tdx_resize_aa_axis(x, 4, 4, o, 8, 2, s),
        "blur even ksize": lambda: lib.tdx_gaussian_blur(x, 16, 16, o, 4, 1.0, s),
        "blur ksize 33": lambda: lib.tdx_gaussian_blur(x, 40, 40, o, 33, 5.0, s),
        "blur h == ksize / 2": lambda: lib.tdx_gaussian_blur(x, 5, 40, o, 11, 5.0, s),
        "blur w == ksize / 2": lambda: lib.tdx_gaussian_blur(x, 40, 1, o, 3, 0.8, s),
        "blur h > 65535": lambda: lib.tdx_gaussian_blur(x, 65536, 1, o, 1, 0.8, s),
        "combine a_pitch < w": lambda: lib.tdx_post_combine(x, 7, x, 8, o, None, 2, 8, 0, s),
        "combine b_pitch < w": lambda: lib.tdx_post_combine(x, 8, x, 7, o, None, 2, 8, 0, s),
        "combine h > 65535": lambda: lib.tdx_post_combine(x, 1, x, 1, o, None, 65536, 1, 0, s),
        "lapse even win": lambda: lib.tdx_lapse_rate(x, x, 16, 16, 4, -0.012, 0.0, -0.0065, 1e-6, 0.3, o, o, s),
        "lapse win 1": lambda: lib.tdx_lapse_rate(x, x, 16, 16, 1, -0.012, 0.0, -0.0065, 1e-6, 0.3, o, o, s),
        "lapse win > h": lambda: lib.tdx_lapse_rate(x, x, 14, 40, 15, -0.012, 0.0, -0.0065, 1e-6, 0.3, o, o, s),
        "lapse win > w": lambda: lib.tdx_lapse_rate(x, x, 40, 14, 15, -0.012, 0.0, -0.0065, 1e-6, 0.3, o, o, s),
        "lapse h > 65535": lambda: lib.tdx_lapse_rate(x, x, 65536, 3, 3, -0.012, 0.0, -0.0065, 1e-6, 0.3, o, o, s),
        "climate n_ch < 6": lambda: lib.tdx_climate_sample(x, x, x, 5, 15, 15, 7, x, 0, 0, 4, 4, 64, 0, 0, o, s),
        "climate hc <= 2 crop": lambda: lib.tdx_climate_sample(x, x, x, 6, 14, 15, 7, x, 0, 0, 4, 4, 64, 0, 0, o, s),
        "climate wc <= 2 crop": lambda: lib.tdx_climate_sample(x, x, x, 6, 15, 14, 7, x, 0, 0, 4, 4, 64, 0, 0, o, s),
        "climate h > 65535": lambda: lib.tdx_climate_sample(x, x, x, 6, 15, 15, 7, x, 0, 0, 65536, 1, 64, 0, 0, o, s),
    }
    prefix = {"post_normalize": b"post_normalize:", "pad": b"post_pad_extrapolate:", "resize": b"resize_aa_axis:",
              "blur": b"gaussian_blur:", "combine": b"post_combine:", "lapse": b"lapse_rate:",
              "climate": b"climate_sample:"}
    for what, call in bad.items():
        assert call() != 0, what
        assert lib.tdx_last_error().startswith(prefix[what.split()[0]]), (what, lib.tdx_last_error())
    torch.cuda.synchronize()
    out.check("rejected launches")
    assert bool(torch.isnan(out.view).all()), "a rejected call wrote its output"
