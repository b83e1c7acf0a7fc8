"""Depression fill and river-bed smoothing, CPU side: the oracle restatement (oracle/depressions.py) against the
golden vectors recorded from the reference's own fill_depressions_priority_flood / smooth_river_bumps
(tests/golden/make_golden_depressions.py), and the argument checks of terrain_diffusion_b200.inference.hydrology.

Tolerances: the fill is bit-identical.  The smoothing's weight is exp in fp64 rounded once here, where numpy uses a
SIMD fp32 exp that is off by up to 2 ulp; after three iterations a pixel may differ from the reference by
SMOOTH_BOUND_ULPS ulps of the window's largest finite |height| (2 observed)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import depressions as O
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import hydrology as H
from tests._depression_inputs import FILL_CASES, SMOOTH_CASES, fill_case, smooth_case

ROOT = Path(__file__).resolve().parent.parent
G = np.load(ROOT / "tests" / "golden" / "depressions_golden.npz")
SMOOTH_BOUND_ULPS = 4


def same_bits(a, b) -> bool:
    return a.dtype == b.dtype == np.float32 and a.shape == b.shape and np.array_equal(a.view(np.uint32),
                                                                                      b.view(np.uint32))


def smooth_within_bound(got, ref, z) -> bool:
    """NaN in the same places; elsewhere within SMOOTH_BOUND_ULPS fp32 ulps of the window's largest finite |z|."""
    nan = np.isnan(ref)
    if got.shape != ref.shape or not np.array_equal(np.isnan(got), nan):
        return False
    scale = np.spacing(np.float32(np.max(np.abs(z[np.isfinite(z)]), initial=1.0)))
    return bool(np.all(np.abs(got[~nan].astype(np.float64) - ref[~nan]) <= SMOOTH_BOUND_ULPS * float(scale)))


@pytest.mark.parametrize("name", list(FILL_CASES))
def test_fill_oracle_matches_reference_golden(name):
    z, kw = fill_case(name)
    out, passes = O.fill(z, **kw)
    assert same_bits(out, G[f"fill.{name}"]) and passes >= 1
    assert same_bits(O.fill_ordered(z, **kw), G[f"fill.{name}"])


@pytest.mark.parametrize("name", list(SMOOTH_CASES))
def test_smooth_oracle_within_bound_of_reference_golden(name):
    z, kw = smooth_case(name)
    got = O.smooth(z, **kw)
    assert got.dtype == np.float32 and smooth_within_bound(got, G[f"smooth.{name}"], z)
    if kw.get("iterations") == 0:
        assert same_bits(got, G[f"smooth.{name}"])


def test_golden_cases_cover_the_branches():
    # pits are raised; epsilon 0 leaves flats flat; the 0.05 case raises by more than the default
    z, _ = fill_case("pits8")
    assert (G["fill.pits8"] > z).sum() > 100 and np.isnan(z).any() and (z < 0).any()
    z, _ = fill_case("plateau_eps0")
    raised = G["fill.plateau_eps0"] > z
    assert raised.any() and np.all(np.isin(G["fill.plateau_eps0"][raised], np.unique(z)))   # filled to a rim level
    z, _ = fill_case("pits_eps005")
    assert float(np.max(G["fill.pits_eps005"] - G["fill.pits8"], where=~np.isnan(z), initial=0)) > 0.01
    # 4- and 8-connectivity differ
    assert not np.array_equal(G["fill.pits4"], G["fill.pits8"], equal_nan=True)
    # nodata pixels keep their value and act as ocean: the cells around them are seeds
    z, kw = fill_case("nodata")
    assert np.all(G["fill.nodata"][z == 7777.0] == 7777.0)
    _, invalid, seed = O.classify(z, 8, kw["nodata"])
    assert invalid[z == 7777.0].all() and seed[29, 10] and seed[33, 10]
    # at 40 000 m the epsilon add rounds away: fl32(m + fl32(1e-3)) == m
    z, _ = fill_case("high")
    assert np.float32(40000.0) + np.float32(1e-3) == np.float32(40000.0) and (G["fill.high"] > z).sum() > 10
    # +inf is land and walls the flood; -inf is ocean
    z, _ = fill_case("inf_land")
    assert np.all(G["fill.inf_land"][np.isposinf(z)] == np.inf) and np.all(G["fill.inf_land"][np.isneginf(z)] == -np.inf)
    # the smoothing NaN cases wrap NaN around the image edges
    z, _ = smooth_case("nan")
    assert np.isnan(z[0]).any() and np.isnan(z[:, -1]).any()
    # routing the filled window drains more land through long paths than the raw one
    assert float(G["compose.A"].max()) > 20


def test_fill_relaxation_counts_passes_of_the_longest_chain():
    # a one-cell-wide flat corridor, entered at one end: every Jacobi pass extends the settled chain by one cell
    z = np.full((3, 40), 500.0, np.float32)
    z[1, 1:-1] = 10.0
    z[1, 0] = 5.0                                            # the only seed below the walls
    out, passes = O.fill(z)
    e = np.float32(1e-3)
    want = [np.float32(5.0), np.float32(10.0)]               # 10 > 5: kept
    for _ in range(2, 39):
        want.append(want[-1] + e)                            # flat: raised by one fp32 epsilon add per cell
    assert np.array_equal(out[1, :39], want) and out[1, 39] == 500.0
    assert passes == 39                                      # 38 cells settled one per pass, then one quiet pass
    assert same_bits(out, O.fill_ordered(z))


def test_argument_errors_come_before_any_device_work(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(L, "lib", no_device)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    fill, smooth = H.fill_depressions_priority_flood, H.smooth_river_bumps
    z = np.full((6, 7), 10.0, np.float32)
    for bad in (np.zeros(5, np.float32), np.zeros((0, 4), np.float32), np.zeros((3, 0), np.float32),
                np.zeros((2, 3, 4), np.float32), np.zeros((6, 7), np.int32), torch.zeros(6, 7, dtype=torch.int64),
                np.zeros((4097, 4096), np.float32), torch.zeros(1, 2 ** 24 + 1)):
        for fn in (fill, smooth):
            with pytest.raises(ValueError):
                fn(bad)
    with pytest.raises(NotImplementedError, match="max_raise"):
        fill(z, max_raise=5.0)
    with pytest.raises(NotImplementedError, match="max_raise"):
        fill(torch.zeros(6, 7, dtype=torch.int64), max_raise=0.0)     # before the input checks
    for eps in (-1e-3, float("nan"), float("inf"), "x", None):
        with pytest.raises(ValueError, match="epsilon"):
            fill(z, epsilon=eps)
    for shape in ((1, 7), (7, 1), (1, 1)):                   # np.gradient needs two samples per axis
        with pytest.raises(ValueError, match="2 rows"):
            smooth(np.ones(shape, np.float32))
    with pytest.raises(ValueError, match="iterations"):
        smooth(z, iterations=2.0)
    zi = z.copy()
    zi[2, 3], zi[4, 4] = np.inf, -np.inf                      # legal here: +inf is land, -inf ocean
    for args in ((fill, z), (fill, zi), (smooth, zi), (fill, np.ones((1, 5), np.float32))):
        with pytest.raises(L.TdxError):                      # valid arguments, no CUDA device
            args[0](args[1])


def test_nodata_is_compared_as_numpy_compares_it():
    assert H._nodata32(None) != H._nodata32(None)            # NaN: matches nothing
    assert H._nodata32(0.1) == float(np.float32(0.1))         # a Python float rounds to fp32
    assert np.isnan(H._nodata32(np.float64(0.1)))             # a float64 scalar fp32 cannot hold matches nothing
    assert H._nodata32(np.float64(0.5)) == 0.5 and H._nodata32(-9999) == -9999.0
    z = np.array([[0.1, 0.5]], np.float32)
    for nd in (0.1, np.float64(0.1), np.float64(0.5), np.float32(0.1)):
        _, invalid, _ = O.classify(z, 8, nd)                 # the oracle compares as the reference does
        assert np.array_equal(invalid[0], z[0] == nd)
        assert np.array_equal(invalid[0], z[0] == np.float32(H._nodata32(nd)))


def test_bench_depressions_help_runs():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_depressions.py"), "--help"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--iters" in out.stdout and "--sizes" in out.stdout and "--serpentine" in out.stdout
