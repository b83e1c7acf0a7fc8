"""River routing, depression fill and river smoothing through their C entry points (csrc/tdx_hydro.cu,
csrc/tdx_depress.cu), with the arguments the Python wrappers never pass.

- Every fp32 output lives in a guarded NaN-filled buffer (tests/_igemm_ref.Guarded), so a stray write or an unwritten
  element fails.  Every integer output is written twice, over a 0x00 and over a 0xFF fill between sentinel guards:
  the two results must agree, so every element is written.  Scratch buffers start filled with garbage, so each call
  must reset what it reads.
- Results are compared bit for bit with oracle/hydrology.py and oracle/depressions.py, which are pinned to the
  reference's goldens (NaN by position).
- tdx_flow_d8 sweeps its 32 x 8 tile and ring on seam-stressing fields and every output combination; tdx_flow_link
  raises each flag alone and together; tdx_flow_accumulate runs forests no D8 field produces; tdx_flow_indicator is
  tested over every integer count up to 2^24; tdx_fill_depressions sweeps its 32 x 32 tile, long chains and its
  parameter edges; tdx_smooth_river_bumps its iteration counts, wrap-around shapes and parameter edges.
- Argument checks get real buffers of the full size, so a missing check shows as a wrong result, not a stray write.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import depressions as OD
from oracle import hydrology as O
from terrain_diffusion_b200 import _lib as L
from tests._igemm_ref import Guarded, report

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
FLOW_INF, FLOW_RANGE, FLOW_NOT_DOWNHILL = 1, 2, 4
FILL_BATCH = 32
GUARD = 256                  # bytes of sentinel on each side of an integer output
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def found(request):
    seen: dict = {}
    yield seen
    report(request.config, [f"{k}: {v}" for k, v in seen.items()])


class IntBuf:
    """An integer tensor between GUARD-byte sentinel guards, its body filled with the byte `fill`."""

    def __init__(self, shape, dtype, fill):
        self.nbytes = int(np.prod(shape, dtype=np.int64)) * torch.empty((), dtype=dtype).element_size()
        self.raw = torch.full((2 * GUARD + self.nbytes,), SENTINEL, dtype=torch.uint8, device=DEV)
        self.raw[GUARD:GUARD + self.nbytes].fill_(fill)
        self.view = self.raw[GUARD:GUARD + self.nbytes].view(dtype).view(*shape)

    def data_ptr(self):
        return self.view.data_ptr()

    def check(self, what):
        bad = int((self.raw[:GUARD] != SENTINEL).sum()) + int((self.raw[GUARD + self.nbytes:] != SENTINEL).sum())
        assert bad == 0, f"{what}: {bad} bytes written outside the tensor"


def garbage(shape, dtype, seed=0):
    """A scratch tensor full of random bytes."""
    n = int(np.prod(shape, dtype=np.int64)) * torch.empty((), dtype=dtype).element_size()
    g = torch.Generator(device=DEV).manual_seed(seed)
    raw = torch.randint(0, 256, (n,), dtype=torch.uint8, device=DEV, generator=g)
    return raw.view(dtype).view(*shape)


def twice(launch, specs):
    """Run launch(bufs) over 0x00- and 0xFF-filled integer outputs {name: (shape, dtype)}: checks the guards and that
    both runs agree, and returns {name: numpy array}."""
    runs = []
    for fill in (0x00, 0xFF):
        bufs = {k: IntBuf(s, d, fill) for k, (s, d) in specs.items()}
        launch(bufs)
        torch.cuda.synchronize()
        for k, b in bufs.items():
            b.check(k)
        runs.append({k: b.view.cpu().numpy().copy() for k, b in bufs.items()})
    for k in specs:
        assert np.array_equal(runs[0][k], runs[1][k]), f"{k}: some elements were not written"
    return runs[1]


def dev(a, dtype=F32):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).to(DEV)


def assert_bits(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ at {int((np.isnan(got) ^ nan).sum())}"
    diff = (got.view(np.uint32) != want.view(np.uint32)) & ~nan
    if diff.any():
        i = tuple(int(v) for v in np.argwhere(diff)[0])
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ; first at {i}: got {got[i]!r}, want {want[i]!r}")


# ---------------------------------------------------------------------------------------------------------------------
# tdx_flow_d8
# ---------------------------------------------------------------------------------------------------------------------
D8_OUTS = ("kmax", "is_sink", "rr", "cc", "recv", "indeg")
D8_TYPES = {"kmax": torch.int8, "is_sink": torch.uint8, "rr": torch.int64, "cc": torch.int64, "recv": torch.int32,
            "indeg": torch.int32}


def run_d8(z, tol=1e-3, outs=D8_OUTS):
    """tdx_flow_d8 with the outputs `outs` (the others NULL) and the flag word: {name: numpy array, 'flags': int}."""
    h, w = z.shape
    zd = dev(z)
    specs = {k: ((h, w), D8_TYPES[k]) for k in outs}
    specs["flags"] = ((1,), torch.int32)

    def launch(b):
        L.call(L.lib().tdx_flow_d8, DEV, zd.data_ptr(), h, w, float(F32(tol)),
               *[b[k].data_ptr() if k in b else None for k in D8_OUTS], b["flags"].data_ptr())

    res = twice(launch, specs)
    res["flags"] = int(res["flags"][0]) & 0xFFFFFFFF
    return res


def d8_reference(z, tol=1e-3):
    rr, cc, is_sink, kmax = O.d8(z, tol)
    recv = O.receivers(z, rr, cc, is_sink)
    indeg = np.bincount(recv[recv >= 0], minlength=z.size)
    return {"kmax": kmax.astype(np.int8), "is_sink": is_sink.astype(np.uint8), "rr": rr, "cc": cc,
            "recv": recv.reshape(z.shape).astype(np.int32), "indeg": indeg.reshape(z.shape).astype(np.int32)}


SEAM_ROWS, SEAM_COLS = (7, 8, 15, 16, 31, 32, 63, 64), (31, 32, 63, 64, 95, 96)


def seam_field(h, w, seed):
    """Elevations on a 0.25 m grid (exact slopes, many exact ties and equal N / W slopes), a plateau straddling the
    first tile corner, and ocean (0, -0, negative, -inf) and NaN on seam rows and columns and in image corners."""
    rng = np.random.RandomState(seed)
    z = (np.float32(1.0) + np.float32(0.25) * rng.randint(0, 6, size=(h, w))).astype(F32)
    z[4:12, 28:36] = F32(1.5)                                  # an exact-tie plateau across both seams
    specials = np.array([0.0, -0.0, -3.0, -np.inf, np.nan], F32)
    for r in SEAM_ROWS:
        if r < h:
            m = rng.rand(w) < 0.15
            z[r, m] = rng.choice(specials, m.sum())
    for c in SEAM_COLS:
        if c < w:
            m = rng.rand(h) < 0.15
            z[m, c] = rng.choice(specials, m.sum())
    for y, x in ((0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)):
        if rng.rand() < 0.5:
            z[y, x] = rng.choice(specials)
    return z


def smooth_small(h, w, seed):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w]
    return (50 + 20 * np.sin(0.3 * y + 0.2 * x + rng.uniform(0, 6)) + rng.randn(h, w)).astype(F32)


@pytest.mark.parametrize("h", [1, 2, 3, 7, 8, 9, 16, 17, 33, 65])
def test_flow_d8_tile_and_ring_sweep(h):
    for w in (1, 2, 31, 32, 33, 63, 64, 65, 97):
        for z in (seam_field(h, w, 1000 * h + w), smooth_small(h, w, 7 * h + w)):
            got, want = run_d8(z), d8_reference(z)
            for k in D8_OUTS:
                assert np.array_equal(got[k], want[k]), (h, w, k)
            assert got["flags"] == 0, (h, w)


def test_seam_fields_have_ties_on_the_seams():
    z = seam_field(17, 65, 3)
    _, _, is_sink, kmax = O.d8(z)
    plateau = ~O.ocean(z) & is_sink
    assert plateau[4:12, 28:36].any()                          # flat sinks on the plateau across the seams
    assert np.isneginf(z).any() and np.isnan(z).any() and (z == 0).any()
    assert (kmax == 0).sum() > 50 and (kmax == 2).sum() > 50   # N and W both chosen


@pytest.mark.parametrize("shape", [(9, 33), (17, 65), (40, 70)])
def test_flow_d8_every_output_combination(shape):
    z = seam_field(*shape, seed=11)
    full = run_d8(z)
    combos = [D8_OUTS, ("kmax", "is_sink", "rr", "cc"), ("recv", "indeg")] + [(k,) for k in D8_OUTS]
    for outs in combos:
        got = run_d8(z, outs=outs)
        assert got["flags"] == 0
        for k in outs:
            assert np.array_equal(got[k], full[k]), (outs, k)


@pytest.mark.parametrize("where", ["interior", "seam", "corner", "all_three"])
def test_flow_d8_flags_positive_infinity(where):
    z = smooth_small(24, 70, 5)
    spots = {"interior": [(3, 10)], "seam": [(7, 31)], "corner": [(23, 69)]}
    spots["all_three"] = [p for v in spots.values() for p in v]
    for y, x in spots[where]:
        z[y, x] = np.inf
    assert run_d8(z)["flags"] == FLOW_INF
    z = smooth_small(24, 70, 5)
    z[3, 10] = z[7, 31] = z[23, 69] = -np.inf                  # -inf is ocean: no flag, and the outputs are exact
    got, want = run_d8(z), d8_reference(z)
    assert got["flags"] == 0 and all(np.array_equal(got[k], want[k]) for k in D8_OUTS)


def test_flow_d8_argument_checks():
    lib = L.lib()
    z = dev(np.ones(4097 * 4096, F32))                         # a real buffer for the too-large shape
    flags = IntBuf((1,), torch.int32, 0xFF)
    bad = [(z.data_ptr(), 0, 4, flags.data_ptr()), (z.data_ptr(), 4, 0, flags.data_ptr()),
           (z.data_ptr(), -1, 4, flags.data_ptr()), (z.data_ptr(), 4097, 4096, flags.data_ptr()),
           (None, 4, 4, flags.data_ptr()), (z.data_ptr(), 4, 4, None)]
    for zp, h, w, fp in bad:
        with pytest.raises(L.TdxError):
            L.call(lib.tdx_flow_d8, DEV, zp, h, w, 1e-3, None, None, None, None, None, None, fp)
    torch.cuda.synchronize()
    flags.check("flags")
    assert int(flags.view[0]) == -1                            # refused before the flag word is reset
    L.call(lib.tdx_flow_d8, DEV, z.data_ptr(), 4096, 4096, 1e-3, None, None, None, None, None, None,
           flags.data_ptr())                                   # exactly 2^24 pixels is allowed
    torch.cuda.synchronize()
    assert int(flags.view[0]) == 0


# ---------------------------------------------------------------------------------------------------------------------
# tdx_flow_link
# ---------------------------------------------------------------------------------------------------------------------
def run_link(z, rr, cc, sink):
    h, w = z.shape
    zd, rd, cd, sd = dev(z), dev(rr, np.int64), dev(cc, np.int64), dev(sink, np.uint8)
    specs = {"recv": ((h, w), torch.int32), "indeg": ((h, w), torch.int32), "flags": ((1,), torch.int32)}

    def launch(b):
        L.call(L.lib().tdx_flow_link, DEV, zd.data_ptr(), rd.data_ptr(), cd.data_ptr(), sd.data_ptr(), h, w,
               b["recv"].data_ptr(), b["indeg"].data_ptr(), b["flags"].data_ptr())

    res = twice(launch, specs)
    res["flags"] = int(res["flags"][0]) & 0xFFFFFFFF
    return res


def link_reference(z, rr, cc, sink):
    """recv, indeg and flags of tdx_flow_link restated: an index outside the image raises RANGE (whatever the
    source); a valid, non-sink source into a valid target is followed if the target is strictly lower, else raises
    NOT_DOWNHILL; +inf anywhere raises INF."""
    h, w = z.shape
    zf = z.ravel()
    rr, cc, sink = np.asarray(rr).ravel(), np.asarray(cc).ravel(), np.asarray(sink).ravel()
    inside = (rr >= 0) & (rr < h) & (cc >= 0) & (cc < w)
    t = np.where(inside, rr * w + cc, 0)
    valid = ~O.ocean(zf)
    follow = inside & valid & (sink == 0) & valid[t]
    down = follow & (zf[t] < zf)
    recv = np.where(down, t, -1)
    flags = (FLOW_INF if np.isposinf(zf).any() else 0) | (FLOW_RANGE if (~inside).any() else 0) | \
        (FLOW_NOT_DOWNHILL if (follow & ~down).any() else 0)
    indeg = np.bincount(recv[recv >= 0], minlength=zf.size)
    return recv.reshape(h, w).astype(np.int32), indeg.reshape(h, w).astype(np.int32), flags


def link_case():
    z = smooth_small(12, 40, 21)
    z[5, 5:9] = np.nan
    z[9, 30:33] = -1.0
    rr, cc, is_sink, _ = O.d8(z)
    sink = is_sink.astype(np.uint8)
    rng = np.random.RandomState(22)
    sink[sink == 1] = rng.randint(1, 256, size=int(sink.sum()))    # any non-zero byte is a sink
    assert (sink >= 2).any()
    return z, rr.copy(), cc.copy(), sink


def check_link(z, rr, cc, sink, flags):
    got = run_link(z, rr, cc, sink)
    recv, indeg, want_flags = link_reference(z, rr, cc, sink)
    assert want_flags == flags
    assert got["flags"] == flags and np.array_equal(got["recv"], recv) and np.array_equal(got["indeg"], indeg)


def test_flow_link_follows_d8_receivers():
    z, rr, cc, sink = link_case()
    check_link(z, rr, cc, sink, 0)
    recv, _, _ = link_reference(z, rr, cc, sink)
    assert np.array_equal(recv.ravel(), O.receivers(z, rr, cc, sink != 0))


def _land_pusher(z, rr, cc, sink, k=0):
    """The k-th valid non-sink pixel whose d8 target is valid: (y, x)."""
    ys, xs = np.nonzero(~O.ocean(z) & (sink == 0) & ~O.ocean(z[rr, cc]))
    return int(ys[k]), int(xs[k])


@pytest.mark.parametrize("bad", ["rr=-1", "rr=h", "cc=w", "cc=-1", "rr=2^32+r", "cc=2^32+c"])
def test_flow_link_range_flag(bad):
    z, rr, cc, sink = link_case()
    h, w = z.shape
    y, x = _land_pusher(z, rr, cc, sink, 3)
    which, value = bad.split("=")
    arr = rr if which == "rr" else cc
    arr[y, x] = {"-1": -1, "h": h, "w": w, "2^32+r": 2 ** 32 + int(rr[y, x]), "2^32+c": 2 ** 32 + int(cc[y, x])}[value]
    check_link(z, rr, cc, sink, FLOW_RANGE)
    sink[y, x] = 1                                             # checked for a sink source too
    check_link(z, rr, cc, sink, FLOW_RANGE)


def test_flow_link_not_downhill_flag():
    for kind in ("level", "uphill"):
        z, rr, cc, sink = link_case()
        y, x = _land_pusher(z, rr, cc, sink, 5)
        ty, tx = int(rr[y, x]), int(cc[y, x])
        z[ty, tx] = z[y, x] if kind == "level" else z[y, x] + F32(1.0)
        sink = np.where(O.ocean(z), np.uint8(1), sink).astype(np.uint8)
        check_link(z, rr, cc, sink, FLOW_NOT_DOWNHILL)


def test_flow_link_inf_flag_and_unchecked_edges():
    z, rr, cc, sink = link_case()
    recv, indeg, _ = link_reference(z, rr, cc, sink)
    leaf = np.flatnonzero((indeg.ravel() == 0) & (recv.ravel() >= 0))[0]
    z.flat[leaf] = np.inf                                      # a +inf leaf draining into lower land: only INF
    check_link(z, rr, cc, sink, FLOW_INF)
    z, rr, cc, sink = link_case()
    z.flat[leaf] = -np.inf                                     # -inf is ocean: no flag
    check_link(z, rr, cc, sink, 0)
    # an ocean source, a sink source and an ocean target, each pointed uphill: none is followed or checked
    z, rr, cc, sink = link_case()
    (y0, x0), (y1, x1), (y2, x2) = (_land_pusher(z, rr, cc, sink, k) for k in (0, 10, 20))
    top = np.unravel_index(np.nanargmax(z), z.shape)
    z[y0, x0] = -2.0
    rr[y0, x0], cc[y0, x0] = top
    sink[y1, x1] = 2
    rr[y1, x1], cc[y1, x1] = top
    z[rr[y2, x2], cc[y2, x2]] = np.nan
    check_link(z, rr, cc, sink, 0)


def test_flow_link_every_flag_together():
    z, rr, cc, sink = link_case()
    y, x = _land_pusher(z, rr, cc, sink, 2)
    rr[y, x] = -1
    y, x = _land_pusher(z, rr, cc, sink, 6)
    z[rr[y, x], cc[y, x]] = z[y, x]
    z[0, 39] = np.inf
    sink = np.where(O.ocean(z), np.uint8(1), sink).astype(np.uint8)
    check_link(z, rr, cc, sink, FLOW_INF | FLOW_RANGE | FLOW_NOT_DOWNHILL)


def test_flow_link_argument_checks():
    z, rr, cc, sink = link_case()
    h, w = z.shape
    t = [dev(z), dev(rr, np.int64), dev(cc, np.int64), dev(sink, np.uint8)]
    recv, indeg, flags = IntBuf((h, w), torch.int32, 0x11), IntBuf((h, w), torch.int32, 0x11), IntBuf((1,), torch.int32, 0x11)
    ptrs = [x.data_ptr() for x in t] + [h, w, recv.data_ptr(), indeg.data_ptr(), flags.data_ptr()]
    for i in (0, 1, 2, 3, 6, 7, 8):
        args = list(ptrs)
        args[i] = None
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_flow_link, DEV, *args)
    for hh, ww in ((0, w), (h, 0), (-h, w), (-h, -w)):
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_flow_link, DEV, *ptrs[:4], hh, ww, *ptrs[6:])
    torch.cuda.synchronize()
    for b in (recv, indeg, flags):
        b.check("link output")
        assert bool((b.view == 0x11111111).all())


# ---------------------------------------------------------------------------------------------------------------------
# tdx_flow_accumulate
# ---------------------------------------------------------------------------------------------------------------------
def run_accumulate(z, recv):
    n = z.size
    valid = ~O.ocean(z)
    assert np.all(recv[~valid] == -1) and np.all(valid[recv[recv >= 0]])   # a forest as tdx.h requires it
    indeg = np.bincount(recv[recv >= 0], minlength=n).astype(np.int32)
    zd, rd, idd = dev(z), dev(recv, np.int32), dev(indeg, np.int32)
    state = garbage((n,), torch.int64, seed=n)
    a = Guarded((n,), torch.float32, DEV)
    L.call(L.lib().tdx_flow_accumulate, DEV, zd.data_ptr(), n, rd.data_ptr(), idd.data_ptr(), state.data_ptr(),
           a.data_ptr())
    torch.cuda.synchronize()
    a.check("A")
    return a.view.cpu().numpy()


def tree_sum(recv, valid, order):
    """A = 1 + the sum over children for valid nodes, 0 for invalid ones, adding children before parents in `order`
    (children first), in int64."""
    a = valid.astype(np.int64)
    r = recv.tolist()
    al = a.tolist()
    for v in order:
        t = r[v]
        if t >= 0:
            al[t] += al[v]
    return np.asarray(al, np.int64)


def test_flow_accumulate_one_root_with_2_24_minus_1_children():
    n = 1 << 24
    z = np.ones(n, F32)
    recv = np.zeros(n, np.int32)
    recv[0] = -1
    a = run_accumulate(z, recv)
    assert a[0] == F32(2 ** 24) and a[0] == 16777216.0 and np.all(a[1:] == 1.0)


def test_flow_accumulate_random_forest_with_lower_parents():
    n = 1 << 20
    rng = np.random.RandomState(31)
    parent = (rng.rand(n) * np.arange(n)).astype(np.int64)      # a parent with a lower index
    root = rng.rand(n) < 0.01
    root[0] = True
    recv = np.where(root, -1, parent)
    # invalid leaves and roots: isolated pixels that are NaN, 0, negative or -inf
    has_child = np.zeros(n, bool)
    has_child[recv[recv >= 0]] = True
    iso = np.flatnonzero(root & ~has_child)[:500].tolist() + np.flatnonzero(~has_child & ~root)[:500].tolist()
    z = np.full(n, 10.0, F32)
    z[iso] = np.resize(np.array([np.nan, 0.0, -0.0, -5.0, -np.inf], F32), len(iso))
    recv[iso] = -1
    has_child = np.zeros(n, bool)
    has_child[recv[recv >= 0]] = True
    assert not has_child[iso].any()
    want = tree_sum(recv, ~O.ocean(z), range(n - 1, -1, -1))
    a = run_accumulate(z, recv.astype(np.int32))
    assert np.array_equal(a, want.astype(F32)) and want.max() > 1000 and np.all(a[iso] == 0)


@pytest.mark.parametrize("layout", ["reversed", "shuffled"])
def test_flow_accumulate_long_chain_against_thread_order(layout):
    n = 1 << 16
    order = np.arange(n)[::-1] if layout == "reversed" else np.random.RandomState(32).permutation(n)
    recv = np.full(n, -1, np.int64)
    recv[order[:-1]] = order[1:]                               # order[0] is the leaf, order[-1] the outlet
    z = np.full(n, 3.0, F32)
    a = run_accumulate(z, recv.astype(np.int32))
    want = np.empty(n, F32)
    want[order] = np.arange(1, n + 1, dtype=F32)
    assert np.array_equal(a, want)


def test_flow_accumulate_argument_checks():
    n = (1 << 24) + 1                                          # real buffers one element past the limit
    z, recv, indeg = dev(np.ones(n, F32)), dev(np.full(n, -1, np.int32), np.int32), dev(np.zeros(n, np.int32), np.int32)
    state = torch.zeros(n, dtype=torch.int64, device=DEV)
    a = Guarded((n,), torch.float32, DEV)
    ptrs = [z.data_ptr(), n, recv.data_ptr(), indeg.data_ptr(), state.data_ptr(), a.data_ptr()]
    for count in (0, -1, n):
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_flow_accumulate, DEV, ptrs[0], count, *ptrs[2:])
    for i in (0, 2, 3, 4, 5):
        args = list(ptrs)
        args[1] = 16
        args[i] = None
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_flow_accumulate, DEV, *args)
    torch.cuda.synchronize()
    a.check("A")
    assert bool(torch.isnan(a.view).all())


# ---------------------------------------------------------------------------------------------------------------------
# tdx_flow_indicator
# ---------------------------------------------------------------------------------------------------------------------
def run_indicator(a, k, out_shape):
    h, w = a.shape
    ad = dev(a)
    out = Guarded(out_shape, torch.float32, DEV)
    L.call(L.lib().tdx_flow_indicator, DEV, ad.data_ptr(), h, w, k, out.data_ptr())
    torch.cuda.synchronize()
    out.check("indicator")
    return out.view.cpu().numpy()


def log1p_excusable(r):
    """fp64 results within 2 fp64 ulps of an fp32 rounding midpoint, where a 1-ulp error of either side's fp64
    log1p may round the other way."""
    f = r.astype(F32)
    other = np.nextafter(f, np.where(r > f.astype(np.float64), F32(np.inf), F32(-np.inf)))
    mid = (f.astype(np.float64) + other.astype(np.float64)) / 2
    return np.abs(r - mid) <= 2 * np.spacing(r)


def test_flow_indicator_every_count_up_to_2_24(found):
    a = np.arange(1 << 24, dtype=F32).reshape(4096, 4096)
    got = run_indicator(a, 1, (4096, 4096))
    r = np.log1p(a.astype(np.float64))
    want = r.astype(F32)
    diff = got.view(np.uint32) != want.view(np.uint32)
    excused = diff & log1p_excusable(r)
    found["log1p excused (0 .. 2^24 - 1)"] = int(excused.sum())
    assert not (diff & ~excused).any(), f"{int((diff & ~excused).sum())} counts differ, first {np.argwhere(diff)[0]}"
    top = run_indicator(np.full((1, 1), 2.0 ** 24, F32), 1, (1, 1))
    r = np.log1p(np.float64(2 ** 24))
    assert top[0, 0] == F32(r) or log1p_excusable(np.array([r]))[0]


@pytest.mark.parametrize("k", [1, 2, 3, "h", "h+1", 0, -3])
def test_flow_indicator_pool_kernels(k):
    h, w = 20, 26
    rng = np.random.RandomState(41)
    a = rng.randint(0, 5000, size=(h, w)).astype(F32)
    a[rng.rand(h, w) < 0.2] = 0
    kk = {"h": h, "h+1": h + 1}.get(k, k)
    ke = max(int(kk), 1)
    shape = (h // ke, w // ke)
    want = O.indicator(a, np.ones((h, w), F32), kk)
    if shape[0] == 0 or shape[1] == 0:
        out = run_indicator(a, kk, (4,))                       # nothing to write: a guarded buffer stays NaN
        assert want.size == 0 and np.isnan(out).all()
        L.call(L.lib().tdx_flow_indicator, DEV, dev(a).data_ptr(), h, w, kk, None)   # out may be NULL
        return
    got = run_indicator(a, kk, shape)
    assert got.shape == want.shape
    pooled = a[:shape[0] * ke, :shape[1] * ke].reshape(shape[0], ke, shape[1], ke).max(axis=(1, 3))
    exact = np.log1p(pooled.astype(np.float64))
    diff = got.view(np.uint32) != exact.astype(F32).view(np.uint32)
    assert not (diff & ~log1p_excusable(exact)).any()


def test_flow_indicator_argument_checks():
    a = dev(np.ones((8, 8), F32))
    out = Guarded((8, 8), torch.float32, DEV)
    for args in ((a.data_ptr(), 0, 8, 1, out.data_ptr()), (a.data_ptr(), 8, -1, 1, out.data_ptr()),
                 (None, 8, 8, 1, out.data_ptr()), (a.data_ptr(), 8, 8, 2, None)):
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_flow_indicator, DEV, *args)
    torch.cuda.synchronize()
    out.check("indicator")
    assert bool(torch.isnan(out.view).all())


# ---------------------------------------------------------------------------------------------------------------------
# tdx_fill_depressions
# ---------------------------------------------------------------------------------------------------------------------
def run_fill(z, eps=1e-3, connectivity=8, nodata=float("nan")):
    """(out, kind, passes) of tdx_fill_depressions: out guarded, kind written twice, flags guarded garbage."""
    h, w = z.shape
    zd = dev(z)
    outs, passes_seen = [], []

    def launch(b):
        out = Guarded((h, w), torch.float32, DEV)
        flags = IntBuf((FILL_BATCH,), torch.int32, 0x00)
        flags.view.copy_(garbage((FILL_BATCH,), torch.int32, seed=h * w))
        passes = C.c_int32(-7)
        L.call(L.lib().tdx_fill_depressions, DEV, zd.data_ptr(), h, w, float(F32(eps)), connectivity, float(nodata),
               out.data_ptr(), b["kind"].data_ptr(), flags.data_ptr(), C.byref(passes))
        torch.cuda.synchronize()
        out.check("fill out")
        flags.check("fill flags")
        outs.append(out.view.cpu().numpy())
        passes_seen.append(passes.value)

    kind = twice(launch, {"kind": ((h, w), torch.uint8)})["kind"]
    assert outs[0].tobytes() == outs[1].tobytes()
    return outs[1], kind, passes_seen


def fill_reference(z, eps=1e-3, connectivity=8, nodata=None):
    out, jacobi = OD.fill(z, eps, connectivity, nodata)
    _, invalid, seed = OD.classify(z, connectivity, nodata)
    kind = np.where(invalid, 2, np.where(seed, 1, 0)).astype(np.uint8)
    return out, kind, jacobi


def pit_field(h, w, seed):
    """Quantised terrain with pits and plateaus straddling the 32-pixel seams, ocean and NaN."""
    rng = np.random.RandomState(seed)
    z = (np.float32(100.0) + np.float32(4.0) * rng.randint(0, 8, size=(h, w))).astype(F32)
    for cy, cx in ((31, 31), (32, 16), (16, 32), (63, 63), (40, 64)):
        if cy < h and cx < w:
            z[max(cy - 2, 0):cy + 2, max(cx - 2, 0):cx + 3] = F32(60.0)           # a pit across a seam
    for cy, cx in ((30, 40), (50, 30)):
        if cy < h and cx < w:
            z[max(cy - 3, 0):cy + 3, max(cx - 3, 0):cx + 3] = F32(120.0)          # a plateau across a seam
    m = rng.rand(h, w) < 0.03
    z[m] = rng.choice(np.array([np.nan, 0.0, -2.0, -np.inf], F32), m.sum())
    return z


@pytest.mark.parametrize("connectivity", [4, 8, 6])
def test_fill_tile_sweep(connectivity, found):
    sizes = (1, 2, 31, 32, 33, 64, 65)
    seen = []
    for h in sizes:
        for w in sizes:
            z = pit_field(h, w, 100 * h + w)
            out, kind, passes = run_fill(z, connectivity=connectivity)
            want, want_kind, jacobi = fill_reference(z, connectivity=4 if connectivity == 4 else 8)
            assert_bits(out, want, (h, w, connectivity))
            assert np.array_equal(kind, want_kind), (h, w)
            for p in passes:
                if h <= 32 and w <= 32:
                    assert p == (2 if (want_kind == 0).any() else 1), (h, w, p)
                else:
                    assert 1 <= p <= jacobi, (h, w, p, jacobi)
            seen += passes
    found[f"fill sweep passes, connectivity {connectivity}"] = (min(seen), max(seen))


def corridor(w):
    """3 x w: a flat 100 m channel along row 1 between 5000 m walls, draining east through the border pixel
    (1, w - 1): every channel pixel is raised by one epsilon per pixel from the outlet, a chain that crosses
    (w - 2) / 32 tile seams against the CTA order."""
    z = np.full((3, w), 5000.0, F32)
    z[1, 1:] = 100.0
    return z


@pytest.mark.parametrize("w", [40, 200, 600, 1500, 4000])
def test_fill_long_chains_end_in_every_batch(w, found):
    z = corridor(w)
    out, _, passes = run_fill(z)
    want = OD.fill_ordered(z)
    assert_bits(out, want, w)
    assert np.all(np.diff(out[1, 1:-1].astype(np.float64)) < 0)   # a strictly falling chain to the outlet
    for p in passes:
        assert 1 <= p <= w + 1
    found[f"fill corridor 3 x {w} passes"] = passes


@pytest.mark.parametrize("case", ["nodata_inf", "nodata_seed_value", "nodata_nan"])
def test_fill_nodata(case):
    z = pit_field(48, 70, 51)
    z[10:14, 20:30] = np.inf
    seed_value = float(z[0, 5])
    nodata = {"nodata_inf": np.inf, "nodata_seed_value": seed_value, "nodata_nan": np.nan}[case]
    out, kind, _ = run_fill(z, nodata=nodata)
    want, want_kind, _ = fill_reference(z, nodata=None if np.isnan(nodata) else nodata)
    assert_bits(out, want, case)
    assert np.array_equal(kind, want_kind)
    if case != "nodata_nan":
        assert (want_kind[z == F32(nodata)] == 2).all()


@pytest.mark.parametrize("eps", [0.0, float(np.float32(1e-45)), 1e-3])
def test_fill_epsilon_edges(eps):
    z = pit_field(40, 44, 61)
    high = (np.float32(40000.0) + np.float32(4.0) * np.round(z / 25)).astype(F32)      # fl32(40000 + 1e-3) == 40000
    high[np.isnan(z)] = np.nan
    for field in (z, high):
        out, kind, _ = run_fill(field, eps=eps)
        want, want_kind, _ = fill_reference(field, eps=eps)
        assert_bits(out, want, eps)
        assert np.array_equal(kind, want_kind)


def test_fill_argument_checks():
    lib = L.lib()
    big = dev(np.ones(4097 * 4096, F32))
    out = Guarded((4097 * 4096,), torch.float32, DEV)
    kind = IntBuf((4097 * 4096,), torch.uint8, 0x33)
    flags = IntBuf((FILL_BATCH,), torch.int32, 0x33)
    passes = C.c_int32(-7)

    def fill(h, w, eps=1e-3, height=big.data_ptr(), o=out.data_ptr(), k=kind.data_ptr(), f=flags.data_ptr()):
        L.call(lib.tdx_fill_depressions, DEV, height, h, w, eps, 8, float("nan"), o, k, f, C.byref(passes))

    for kw in ({"o": big.data_ptr()}, {"eps": -1e-3}, {"eps": float("inf")}, {"eps": float("nan")},
               {"eps": -float("inf")}, {"height": None}, {"o": None}, {"k": None}, {"f": None}):
        with pytest.raises(L.TdxError):
            fill(64, 64, **kw)
    for h, w in ((4097, 4096), (0, 5), (5, 0), (-1, 5)):
        with pytest.raises(L.TdxError):
            fill(h, w)
    torch.cuda.synchronize()
    out.check("out")
    kind.check("kind")
    flags.check("flags")
    assert bool(torch.isnan(out.view).all()) and bool((kind.view == 0x33).all()) and passes.value == -7


# ---------------------------------------------------------------------------------------------------------------------
# tdx_smooth_river_bumps
# ---------------------------------------------------------------------------------------------------------------------
def run_smooth(z, thresh=50.0, strength=0.3, iterations=3, scratch=True):
    h, w = z.shape
    zd = dev(z)
    out = Guarded((h, w), torch.float32, DEV)
    sc = Guarded((h, w), torch.float32, DEV) if scratch else None
    if sc is not None:
        sc.view.copy_(garbage((h, w), torch.float32, seed=h + w))
    L.call(L.lib().tdx_smooth_river_bumps, DEV, zd.data_ptr(), h, w, float(F32(thresh)), float(F32(strength)),
           iterations, out.data_ptr(), None if sc is None else sc.data_ptr())
    torch.cuda.synchronize()
    out.check("smooth out")
    if sc is not None:
        sc.check("smooth scratch")
    return out.view.cpu().numpy()


def smooth_field_nan(h, w, seed):
    rng = np.random.RandomState(seed)
    z = (300 + 200 * rng.rand(h, w)).astype(F32)
    z[h // 4:h // 2 + 1, w // 4:w // 2 + 1] = F32(250.0)     # a flat patch: zero slope
    z[rng.rand(h, w) < 0.1] = np.nan
    return z


@pytest.mark.parametrize("iterations", [0, 1, 2, 3, 4, 5])
def test_smooth_iterations(iterations):
    z = smooth_field_nan(33, 70, 71)
    assert_bits(run_smooth(z, iterations=iterations), OD.smooth(z, iterations=iterations), iterations)
    if iterations == 1:
        assert_bits(run_smooth(z, iterations=1, scratch=False), OD.smooth(z, iterations=1), "no scratch")


@pytest.mark.parametrize("shape", [(2, 2), (2, 37), (37, 2), (2, 300), (300, 2)])
def test_smooth_wrap_around_shapes(shape):
    z = smooth_field_nan(*shape, seed=shape[0] * 1000 + shape[1])
    assert_bits(run_smooth(z), OD.smooth(z), shape)


@pytest.mark.parametrize("thresh,strength", [(0.0, 0.3), (np.inf, 0.3), (50.0, -0.4), (7.0, 0.45)])
def test_smooth_parameter_edges(thresh, strength):
    z = smooth_field_nan(24, 40, 81)
    want = OD.smooth(z, thresh, strength, 2)
    if thresh == 0:
        assert np.isnan(want).sum() > np.isnan(z).sum()        # 0 / 0 on flat pixels is NaN, as in numpy
    assert_bits(run_smooth(z, thresh, strength, 2), want, (thresh, strength))


def test_smooth_argument_checks():
    h, w = 16, 20
    zd = dev(smooth_field_nan(h, w, 91))
    out = Guarded((h, w), torch.float32, DEV)
    sc = Guarded((h, w), torch.float32, DEV)
    z, o, s = zd.data_ptr(), out.data_ptr(), sc.data_ptr()
    for args in ((z, h, w, 3, z, s), (z, h, w, 3, o, z), (z, h, w, 3, o, o), (z, h, w, 2, o, None),
                 (None, h, w, 1, o, s), (z, h, w, 1, None, s), (z, 1, w, 1, o, s), (z, h, 1, 1, o, s)):
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_smooth_river_bumps, DEV, args[0], args[1], args[2], 50.0, 0.3, args[3], args[4],
                   args[5])
    torch.cuda.synchronize()
    for g in (out, sc):
        g.check("smooth")
        assert bool(torch.isnan(g.view).all())
