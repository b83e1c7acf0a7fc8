"""`coarse_pooling` on the device: `tdx_coarse_epilogue` bit for bit against the reference's own code and the oracle,
the pooled coarse stage against the reference's `_coarse_inference`, and the pooled `WorldPipeline` / `TerrainPipeline`
canvases against directly computed stage windows."""
import json

import numpy as np
import pytest
import torch

from oracle import coarse_pool as O
from oracle import unet as ounet
from terrain_diffusion_b200.inference import (TerrainPipeline, WorldPipeline, coarse_epilogue, coarse_geometry,
                                              coarse_stage_tile)
from terrain_diffusion_b200.inference.stages import pack_weighted
from terrain_diffusion_b200.inference.tiling import linear_weight_window, window_range
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests._coarse_pool_inputs import (GOLDEN, MODES, POOL_SIZES, STAGE_CASES, STAGE_CTX, UNKNOWN_MODES, assert_same,
                                       epilogue_input, golden_epilogue)
from tests._stage_inputs import SEED, stage_inputs
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

G = np.load(GOLDEN)
PAIRS = [(e, p) for e in MODES for p in MODES] + [UNKNOWN_MODES]
TOL = 1.0e-2                                                     # tests/test_stages_gpu.py's stage tolerance


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def build(cfg):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
    return m


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("n", POOL_SIZES)
def test_epilogue_kernel_is_bit_exact_to_the_reference_and_the_oracle(n):
    x, means, stds = epilogue_input()
    ww = linear_weight_window(64 // n)
    batch = torch.stack([x, x.flip(-1), x.transpose(-1, -2), x])                         # n_img = 4
    dev = torch.device("cuda")
    for e, p in PAIRS:
        out = coarse_epilogue(batch.to(dev).contiguous(), means.to(dev), stds.to(dev), ww.to(dev), n, e, p)
        assert out.shape == (4, 7, 64 // n, 64 // n)
        want = golden_epilogue(G, n, e, p) if n > 1 or (e, p) == ("avg", "avg") else golden_epilogue(G, 1, "avg", "avg")
        assert_same(out[0], want, (n, e, p, 0))
        assert_same(out[3], want, (n, e, p, 3))
        for k in (1, 2):
            assert_same(out[k], O.epilogue(batch[k].clone(), means, stds, ww, n, e, p), (n, e, p, k))


def test_epilogue_kernel_at_n1_equals_the_torch_op_sequence_it_replaces():
    """pool_size = 1 keeps today's coarse tiles bit for bit: the de-normalisation, the channel-1 difference and
    pack_weighted as separate CUDA torch ops (torch multiplies by 1 / sigma_data, exact for 0.5)."""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(5)
    raw = torch.randn(3, 6, 64, 64, generator=g) * 3
    x, means, stds = epilogue_input()
    ww = linear_weight_window(64, dev)
    for k, (sample, mu, sd) in enumerate(((raw, torch.randn(6, generator=g), torch.rand(6, generator=g) + 0.5),
                                          (x[None], means, stds))):
        sample, mu, sd = sample.to(dev), mu.to(dev), sd.to(dev)
        old = sample / 0.5 * sd.view(1, -1, 1, 1) + mu.view(1, -1, 1, 1)
        old[:, 1] = old[:, 0] - old[:, 1]
        old = pack_weighted(old.contiguous(), ww)
        new = coarse_epilogue(sample.contiguous(), mu, sd, ww, 1, "max", "min")
        assert_same(new, old.cpu(), k)
        if k == 0:                                                    # no NaN: every bit, sign of zero included
            assert torch.equal(new.view(torch.int32), old.view(torch.int32))


def test_epilogue_rejects_mismatched_arguments():
    dev = torch.device("cuda")
    s = torch.zeros(1, 6, 64, 64, device=dev)
    v6 = torch.ones(6, device=dev)
    with pytest.raises(ValueError, match="window"):
        coarse_epilogue(s, v6, v6, linear_weight_window(64, dev), 2)
    with pytest.raises(ValueError, match="sample"):
        coarse_epilogue(s[:, :5].contiguous(), v6, v6, linear_weight_window(64, dev), 1)
    with pytest.raises(ValueError, match="coarse_pooling"):
        coarse_epilogue(s, v6, v6, linear_weight_window(64, dev), 3)


# ------------------------------------------------------------------------------------------------ the stage
@pytest.mark.parametrize("n,elev,p5", STAGE_CASES)
def test_pooled_coarse_stage_matches_reference_method(n, elev, p5):
    inp = stage_inputs()
    m = build(COARSE_CFG).cuda()
    t_cond = torch.atan(inp["cond_snr"])
    cond_inputs = [v.view(-1) for v in torch.log(torch.tan(t_cond) / 8.0)]
    got = coarse_stage_tile(m, EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5), SEED,
                            STAGE_CTX, inp["coarse_map"].clone(), t_cond, cond_inputs, linear_weight_window(64 // n),
                            inp["coarse_means"].tolist(), inp["coarse_stds"].tolist(), pool_size=n,
                            elev_pool_mode=elev, p5_pool_mode=p5).cpu()
    want = torch.from_numpy(G[f"stage_n{n}_{elev}_{p5}"])
    assert got.shape == want.shape == (7, 64 // n, 64 // n)
    assert torch.equal(got[-1], want[-1])                       # blend weights: bit-exact
    assert rel_rms(got[:-1], want[:-1]) < TOL


# ------------------------------------------------------------------------------------------------ the pipelines
def _cond_fn(i1, i2, j1, j2):
    gg = torch.Generator().manual_seed(i1 * 7919 + j1 + 12345)
    return torch.randn(5, i2 - i1, j2 - j1, generator=gg)


KW = dict(decoder_tile_size=128, decoder_tile_stride=96, residual_mean=0.1, residual_std=1.2, conditioning_fn=_cond_fn)


@pytest.fixture(scope="module")
def models():
    return build(COARSE_CFG).cuda(), build(BASE_CFG).cuda(), build(ounet.DECODER_CFG).cuda()


def _direct_coarse(world, a, b, c, d, n, elev, p5):
    """The coarse canvas over pooled cells [a, b) x [c, d) from coarse_stage_tile windows, summed row-major."""
    tile, stride = coarse_geometry(n)
    sched = EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)
    ww = linear_weight_window(tile, "cuda")
    out = torch.zeros(7, b - a, d - c, device="cuda")
    for i in window_range(a, b, tile, stride, 0):
        for j in window_range(c, d, tile, stride, 0):
            smap = world._conditioning_model_input(i * 48, i * 48 + 64, j * 48, j * 48 + 64)
            t = coarse_stage_tile(world.coarse_model, sched, world.seed, (0, i, j), smap, world._t_cond,
                                  world._cond_inputs, ww, world.kwargs["coarse_means"], world.kwargs["coarse_stds"],
                                  pool_size=n, elev_pool_mode=elev, p5_pool_mode=p5)
            y0, x0 = i * stride, j * stride
            ys, ye, xs, xe = max(a, y0), min(b, y0 + tile), max(c, x0), min(d, x0 + tile)
            out[:, ys - a:ye - a, xs - c:xe - c] += t[:, ys - y0:ye - y0, xs - x0:xe - x0]
    return out.cpu()


def test_pooled_world_pipeline_canvas_get_terrain_pipeline_and_round_trip(models, tmp_path):
    coarse, base, dec = models
    world = WorldPipeline.from_local_models(coarse, base, dec, seed=5, coarse_pooling=2, elev_coarse_pool_mode="max",
                                            p5_coarse_pool_mode="min", **KW).to("cuda").bind()
    # rows 20:30 meet windows 0 and 1 (tile 32, stride 24), columns -10:5 windows -1 and 0
    got = world.coarse[:, 20:30, -10:5]
    assert got.device.type == "cpu" and got.shape == (7, 10, 15)
    assert torch.equal(got, _direct_coarse(world, 20, 30, -10, 5, 2, "max", "min"))
    assert world._coarse.windows_computed == 4
    # the pooling changes the tiles: the same window without it is a different (64^2) tile
    plain = WorldPipeline.from_local_models(coarse, base, dec, seed=5, **KW).to("cuda").bind()
    assert not torch.equal(plain.coarse[:, 20:30, -10:5], got)

    out = world.get(-30, 10, 34, 106, with_climate=True)
    assert out["elev"].device.type == "cpu" and out["elev"].shape == (64, 96) and out["elev"].dtype == torch.float32
    assert out["climate"].shape == (5, 64, 96) and out["climate"].dtype == torch.float32
    assert torch.isfinite(out["elev"]).all() and torch.isfinite(out["climate"]).all()

    ref = TerrainPipeline(coarse, base, dec, seed=5, conditioning_fn=_cond_fn,
                          coarse_means=world.kwargs["coarse_means"], coarse_stds=world.kwargs["coarse_stds"],
                          cond_snr=world.kwargs["cond_snr"], histogram_raw=world.kwargs["histogram_raw"],
                          latents_means=world.cond_input_mean, latents_stds=world.cond_input_std,
                          decoder_tile_size=128, decoder_tile_stride=96, residual_mean=0.1, residual_std=1.2,
                          coarse_pooling=2, elev_coarse_pool_mode="max", p5_coarse_pool_mode="min")
    ref_out = ref.get(-30, 10, 34, 106, with_climate=True)
    assert ref_out["elev"].is_cuda
    assert torch.equal(ref_out["elev"].cpu(), out["elev"]) and torch.equal(ref_out["climate"].cpu(), out["climate"])
    assert torch.equal(ref.coarse[:, 20:30, -10:5].cpu(), got)

    world.save_pretrained(tmp_path / "pooled")
    cfg = json.loads((tmp_path / "pooled" / "config.json").read_text())
    assert (cfg["coarse_pooling"], cfg["elev_coarse_pool_mode"], cfg["p5_coarse_pool_mode"]) == (2, "max", "min")
    back = WorldPipeline.from_pretrained(str(tmp_path / "pooled"), seed=5, conditioning_fn=_cond_fn).to("cuda").bind()
    assert back.kwargs["coarse_pooling"] == 2
    assert torch.equal(back.coarse[:, 20:30, -10:5], got)
    # an unpooled config with the pooling given as keyword arguments, as the generate CLI's --kwarg passes it
    plain.save_pretrained(tmp_path / "plain")
    kw = WorldPipeline.from_pretrained(str(tmp_path / "plain"), seed=5, coarse_pooling=2, elev_coarse_pool_mode="max",
                                       p5_coarse_pool_mode="min", conditioning_fn=_cond_fn).to("cuda").bind()
    out_kw = kw.get(-30, 10, 34, 106)
    assert torch.equal(out_kw["elev"], out["elev"]) and torch.equal(out_kw["climate"], out["climate"])


def test_pool_16_runs_through_get(models):
    """coarse_pooling = 16: 4 x 4 coarse windows at a stride of 3, so each latent window's 4 x 4 coarse read meets
    up to four coarse windows per axis."""
    coarse, base, dec = models
    world = WorldPipeline.from_local_models(coarse, base, dec, seed=9, coarse_pooling=16, elev_coarse_pool_mode="min",
                                            p5_coarse_pool_mode="max", **KW).to("cuda").bind()
    assert world._coarse.win.size[1:] == (4, 4) and world._coarse.win.stride[1:] == (3, 3)
    out = world.get(0, 0, 64, 64)
    assert out["elev"].shape == (64, 64) and out["climate"].shape == (5, 64, 64)
    assert torch.isfinite(out["elev"]).all() and torch.isfinite(out["climate"]).all()
    c = world.coarse[:, -2:7, -2:7]
    assert c.shape == (7, 9, 9) and torch.isfinite(c).all() and float(c[-1].min()) > 0
    assert torch.equal(c, _direct_coarse(world, -2, 7, -2, 7, 16, "min", "max"))
