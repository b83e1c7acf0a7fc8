"""Deterministic inputs shared by tests/golden/make_golden_coarse_pool.py (reference side) and the coarse-pooling tests."""
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden" / "coarse_pool_golden.npz"

POOL_SIZES = (1, 2, 4, 8, 16)
MODES = ("avg", "max", "min")
SIGMA_DATA = 0.5
# the pooled stage cases: (coarse_pooling, elev_coarse_pool_mode, p5_coarse_pool_mode), all at window (0, 1, -2)
STAGE_CASES = ((2, "max", "min"), (4, "avg", "avg"), (16, "min", "max"))
STAGE_CTX = (0, 1, -2)
# mode strings the reference's _pool_channel does not name: they average
UNKNOWN_MODES = ("median", "Max")


def epilogue_input():
    """(x [6, 64, 64] raw solve output, means [6], stds [6]).  The de-normalised channels hold every case the pooling
    arithmetic distinguishes: ties (the left half is on a 0.5 grid), a 16 x 16 block of -0 / +0 (means of -0 keep the
    sign through `* std + mean` in channels 0, 1, 3 and 5), scattered NaN and +-inf, and blocks that are all -inf or
    all NaN in channel 0; channel 1 (= ch0 - ch1) also gets inf - inf."""
    g = torch.Generator().manual_seed(4242)
    x = torch.randn(6, 64, 64, generator=g)
    x[:, :, :32] = torch.round(x[:, :, :32] * 2) / 2
    zeros = torch.where(torch.rand(6, 16, 16, generator=g) < 0.5, -0.0, 0.0)
    x[:, 0:16, 32:48] = zeros
    flat = x.view(6, -1)
    for value in (float("nan"), float("inf"), float("-inf")):
        idx = torch.randint(0, 64 * 64, (6, 24), generator=g)
        flat.scatter_(1, idx, value)
    x[0, 48:52, 0:4] = float("-inf")
    x[0, 52:56, 4:8] = float("nan")
    x[0:2, 60, 60] = float("inf")
    means = torch.tensor([-0.0, -0.0, 0.25, -0.0, 1.5, -0.0])
    stds = torch.rand(6, generator=g) + 0.5
    return x, means, stds


def golden_epilogue(G, n: int, elev_mode: str, p5_mode: str) -> np.ndarray:
    """The reference's packed [7, 64/n, 64/n] tile of epilogue_input() (n = 1 ignores the modes)."""
    key = f"epi_n{n}_{elev_mode}_{p5_mode}" if n > 1 else "epi_n1_avg_avg"
    return np.concatenate([G[key], G[f"epi_n{n}_rest"]])


def assert_same(got, want, what=""):
    """Bit-identical fp32, NaN compared by position (a device NaN and an x86 NaN differ in sign and payload bits)."""
    got = np.ascontiguousarray(torch.as_tensor(got).cpu().numpy(), dtype=np.float32)
    want = np.ascontiguousarray(np.asarray(want), dtype=np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert (gn == wn).all(), (what, "NaN positions differ", int((gn != wn).sum()))
    diff = got[~gn].view(np.uint32) != want[~wn].view(np.uint32)
    assert not diff.any(), (what, f"{int(diff.sum())} values differ", got[~gn][diff][:4], want[~wn][diff][:4])
