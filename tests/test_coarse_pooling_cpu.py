"""`coarse_pooling` without a GPU: argument validation before any device work, the pooled canvas geometry, and the
oracle of the coarse epilogue (oracle/coarse_pool.py) against the reference's own code (coarse_pool_golden.npz)."""
import json

import numpy as np
import pytest
import torch

from oracle import coarse_pool as O
from terrain_diffusion_b200.inference import TerrainPipeline, WorldPipeline, coarse_geometry, coarse_stage_tile
from terrain_diffusion_b200.inference.stages import COARSE_POOL_SIZES, pool_mode_flag
from tests._coarse_pool_inputs import (GOLDEN, MODES, POOL_SIZES, UNKNOWN_MODES, assert_same, epilogue_input,
                                       golden_epilogue)

G = np.load(GOLDEN)
BAD = [0, -2, 3, 12, 32, 2.5]


@pytest.mark.parametrize("bad", BAD)
def test_constructor_rejects_illegal_coarse_pooling_before_any_device_work(bad, tmp_path):
    with pytest.raises(ValueError, match=r"coarse_pooling .*\[1, 2, 4, 8, 16\]"):
        WorldPipeline(coarse_pooling=bad)
    # TerrainPipeline validates before it touches its (here absent) models
    with pytest.raises(ValueError, match="coarse_pooling"):
        TerrainPipeline(None, None, None, seed=1, conditioning_fn=None, coarse_means=[0.0] * 6,
                        coarse_stds=[1.0] * 6, cond_snr=[1.0] * 5, histogram_raw=[0.0] * 5,
                        latents_means=[0.0] * 7, latents_stds=[1.0] * 7, coarse_pooling=bad)
    # a pipeline config carrying it fails before any model folder is read (there is none here)
    (tmp_path / "config.json").write_text(json.dumps({"coarse_pooling": bad}))
    with pytest.raises(ValueError, match="coarse_pooling"):
        WorldPipeline.from_pretrained(str(tmp_path))
    with pytest.raises(ValueError, match="coarse_pooling"):
        coarse_stage_tile(None, None, 0, (0, 0, 0), None, None, None, None, None, None, pool_size=bad)


@pytest.mark.parametrize("n", POOL_SIZES)
def test_geometry_of_every_legal_pool_size(n):
    tile, stride = coarse_geometry(n)
    assert (tile, stride) == (64 // n, 48 // n) and tile * n == 64 and stride * n == 48
    # window i of the pooled canvas is the solve at conditioning cell 48 i, the reference's i * (48 // n) * n
    assert all(i * stride * n == i * (48 // n) * n == 48 * i for i in range(-3, 4))
    assert coarse_geometry(np.int64(n)) == (tile, stride)
    p = WorldPipeline(coarse_pooling=np.int64(n), elev_coarse_pool_mode="max", p5_coarse_pool_mode="min")
    assert type(p.kwargs["coarse_pooling"]) is int and p.kwargs["coarse_pooling"] == n
    assert (p.kwargs["elev_coarse_pool_mode"], p.kwargs["p5_coarse_pool_mode"]) == ("max", "min")
    json.dumps(p.kwargs)                                       # save_pretrained writes them as they are


def test_legal_pool_sizes_are_the_common_divisors_of_tile_and_stride():
    assert COARSE_POOL_SIZES == POOL_SIZES == (1, 2, 4, 8, 16)


@pytest.mark.parametrize("n", POOL_SIZES)
def test_oracle_is_bit_exact_to_the_reference_epilogue(n):
    x, means, stds = epilogue_input()
    assert np.array_equal(G["epi_means"].view(np.uint32), means.numpy().view(np.uint32))
    assert np.array_equal(G["epi_stds"].view(np.uint32), stds.numpy().view(np.uint32))
    from terrain_diffusion_b200.inference.tiling import linear_weight_window
    ww = linear_weight_window(64 // n)
    pairs = [(e, p) for e in MODES for p in MODES]
    for e, p in pairs:
        got = O.epilogue(x.clone(), means, stds, ww, n, e, p)
        assert_same(got, golden_epilogue(G, n, e, p), (n, e, p))
    if n > 1:
        assert_same(O.epilogue(x.clone(), means, stds, ww, n, *UNKNOWN_MODES),
                    golden_epilogue(G, n, *UNKNOWN_MODES), (n, UNKNOWN_MODES))


def test_epilogue_inputs_reach_every_pooling_case():
    """The golden input exercises what the arithmetic distinguishes: NaN and inf in the pooled windows, -0 next to +0,
    and ties; otherwise the bit-exact comparisons above would prove less than they claim."""
    x, means, stds = epilogue_input()
    v = x / 0.5 * stds.view(-1, 1, 1) + means.view(-1, 1, 1)
    v[1] = v[0] - v[1]
    for c in (0, 1):
        ch = v[c]
        assert torch.isnan(ch).any() and torch.isposinf(ch).any() and torch.isneginf(ch).any()
        zeros = ch[0:16, 32:48][ch[0:16, 32:48] == 0]
        assert zeros.numel() > 200 and torch.signbit(zeros).any() and (~torch.signbit(zeros)).any()
        cells = ch[:, :32].reshape(32, 2, 16, 2).permute(0, 2, 1, 3).reshape(32, 16, 4)
        top = cells.max(dim=-1, keepdim=True).values
        assert int(((cells == top).sum(-1) > 1).sum()) >= 10               # 2x2 windows whose maximum is tied


def test_unknown_mode_string_means_avg():
    assert [pool_mode_flag(m) for m in ("avg", "max", "min", "median", "Max", "", None, 1)] == [0, 1, 2, 0, 0, 0, 0, 0]
    for n in POOL_SIZES[1:]:
        assert_same(golden_epilogue(G, n, *UNKNOWN_MODES), golden_epilogue(G, n, "avg", "avg"), n)
