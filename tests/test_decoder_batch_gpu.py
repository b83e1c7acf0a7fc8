"""The batched decoder stage on the GPU: every window of `decoder_stage_tiles` is bit-identical to `decoder_stage_tile`
of the same window, and a world built with a larger `decoder_batch_size` to one built with 1.

- the planner gives every launch of the decoder the same (N, ksplit) at every padded batch in batch-invariant mode, at
  128^2 and 512^2, and those launches, replayed at the padded batch sizes, match the fp64 reference
  (tests/_igemm_ref.py);
- random window sets (negative and non-contiguous indices) at every batch size, one and two consistency steps, host and
  device latent windows, and once on 512^2 windows;
- the noise drawn inside a batch is the one-window noise, and a NaN latent window gives the same bits batched and alone;
- world.residual, get() with and without climate and get_terrain(scale=2) of worlds with the two largest
  decoder_batch_size against 1, cold and after empty_cache(), in two request orders (each order against a world with
  decoder_batch_size 1 that saw the same requests);
- torch_compile=True builds the batched decoder programs in bind().
"""
from __future__ import annotations

import ctypes as C
import math
import random

import pytest
import torch

from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import WorldPipeline, pipeline, samplers, stages
from terrain_diffusion_b200.inference.noise import gaussian_noise_patch
from terrain_diffusion_b200.inference.samplers import _solve_cache
from terrain_diffusion_b200.inference.stages import DECODER_BATCH_SIZES, decoder_stage_tile, decoder_stage_tiles
from terrain_diffusion_b200.inference.tiling import linear_weight_window
from terrain_diffusion_b200.models import EDMUnet2D
from tests import _igemm_ref as IR
from tests.test_decoder_batch_cpu import recorded
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

SEED = 20261018
TILE, STRIDE = 128, 96
T_INIT = math.atan(80.0 / 0.5)                   # WorldPipeline.t_init: the product's one decoder step
TWO_STEPS = [T_INIT, math.atan(0.35 / 0.5)]
TOP = DECODER_BATCH_SIZES[-1]


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def build(cfg):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
    return m


@pytest.fixture(scope="module")
def decoder():
    return build(ounet.DECODER_CFG).cuda()


# ------------------------------------------------------------------------------------------------ the planner
@pytest.mark.parametrize("hw", [TILE, 512])
def test_batch_invariant_plans_keep_the_one_window_shape_on_this_gpu(request, hw):
    """(N, ksplit) of every launch of the decoder forward: the one-window plan's at every padded batch, with this GPU's
    SM count and cluster occupancy.  The split-K launches are written to the terminal."""
    plain = [L.igemm_launch_shape(d) for d in recorded(1, hw, False)]
    for n in DECODER_BATCH_SIZES:
        assert [L.igemm_launch_shape(d) for d in recorded(n, hw, True)] == plain, n
    split = [(int(d.height), int(d.c_out), s) for d, s in zip(recorded(1, hw, False), plain) if s[1] > 1]
    IR.report(request.config, [f"decoder forward at {hw}^2: {len(plain)} igemm launches, split-K "
                               f"(h, c_out, (N, ksplit)): {split}"])


def _replay_cases():
    """One launch per (layer shape, epilogue, forced shape) of the batch-invariant decoder forward at every padded batch
    size.  At 512^2 only the launches whose forced (N, ksplit) differs from the free plan at that batch: the others are
    the free launches the product-surface replay (tests/test_igemm_plans_gpu.py) already covers at every batch."""
    out, seen = [], set()
    for hw in (TILE, 512):
        for n in DECODER_BATCH_SIZES:
            free = recorded(n, hw, False)
            for d, f in zip(recorded(n, hw, True), free):
                if hw == 512 and (int(d.n_per_item), int(d.ksplit)) == L.igemm_launch_shape(f):
                    continue
                case = IR.case_from_desc(d, name=f"decoder_invariant_{hw}_b{n}", seed=n)
                key = (hw, n, tuple(case.segs), case.h, case.epi, tuple(case.outs), case.resid_pnorm, case.rms_out,
                       case.resid_inv, int(d.ksplit), case.n_item)
                if key not in seen:
                    seen.add(key)
                    case.name += f":{len(seen)}-ks{int(d.ksplit)}"
                    out.append((case, int(d.ksplit)))
    return out


@pytest.mark.parametrize("case,ksplit", _replay_cases(), ids=lambda v: v.name if isinstance(v, IR.Case) else str(v))
def test_batch_invariant_decoder_plans_match_fp64_reference(case, ksplit):
    """IR.check_case with the launch's forced split-K factor."""
    dev = torch.device("cuda:0")
    acts, wts, cvec, resid = IR.make_inputs(case, dev)
    refs = IR.reference(case, acts, wts, cvec, resid)

    def place(name, value):
        if name == "desc":
            value.ksplit = ksplit
            return C.byref(value)
        return value

    gots = IR.run_cuda(case, acts, wts, cvec, resid, place=place)
    for i, (g, r) in enumerate(zip(gots, refs)):
        what = f"{case.name} {'rms_out' if i == len(case.outs) else f'out{i}'}"
        assert not torch.isnan(g).any(), f"{what}: unwritten (NaN) elements"
        if i < len(case.outs):
            assert IR.rel_rms(g, r.bfloat16().double()) < 2e-3, what
        ratio = IR.elementwise_ratio(g, r)
        assert ratio <= 1.0, f"{what}: error {ratio:.2f}x the per-element bound"


# ------------------------------------------------------------------------------------------------ the stage
def _latents(ctxs, tile=TILE, device="cpu"):
    """Packed [6, tile/8, tile/8] latent windows (x w, w) per window, seeded by the window index; on the device they
    are non-contiguous views of a larger tensor."""
    out = []
    s = tile // 8
    for _, i, j in ctxs:
        g = torch.Generator().manual_seed((i * 7919 + j) & 0xFFFFFFFF)
        big = torch.randn(6, s + 3, s + 5, generator=g) * 0.6
        big[5] = torch.rand(s + 3, s + 5, generator=g) + 0.5
        big[:5] *= big[5:]
        out.append(big.to(device)[:, 2:2 + s, 3:3 + s] if device != "cpu" else big[:, 2:2 + s, 3:3 + s].clone())
    return out


def _windows(rng, n):
    """n distinct, scattered window indices, negative ones included."""
    picked = set()
    while len(picked) < n:
        picked.add((rng.randint(-40, 40), rng.randint(-40, 40)))
    return [(0, i, j) for i, j in sorted(picked, key=lambda _: rng.random())]


def _one(model, ctx, lat, t_list, tile=TILE):
    return decoder_stage_tile(model, SEED, ctx, lat, linear_weight_window(tile, "cuda"), t_list, tile, tile * 3 // 4)


def _many(model, ctxs, lats, t_list, tile=TILE):
    return decoder_stage_tiles(model, SEED, ctxs, lats, linear_weight_window(tile, "cuda"), t_list, tile,
                               tile * 3 // 4)


@pytest.mark.parametrize("device", ["cpu", "cuda"])
@pytest.mark.parametrize("steps", [1, 2])
def test_every_batch_size_is_bit_identical_to_one_window_solves(decoder, steps, device):
    """Random window sets at every batch size 1..TOP (the padded sizes unpadded, the others padded)."""
    t_list = [T_INIT] if steps == 1 else TWO_STEPS
    rng = random.Random(steps * 10 + (device == "cuda"))
    for n in range(1, TOP + 1):
        ctxs = _windows(rng, n)
        lats = _latents(ctxs, device=device)
        got = _many(decoder, ctxs, lats, t_list)
        assert len(got) == n and got[0].shape == (2, TILE, TILE)
        assert all(g.data_ptr() == got[0].data_ptr() + k * got[0].numel() * 4 for k, g in enumerate(got))
        for k, (ctx, lat) in enumerate(zip(ctxs, lats)):
            assert same(got[k], _one(decoder, ctx, lat, t_list)), (n, k, ctx)


def test_a_window_keeps_its_bits_in_any_batch(decoder):
    """The same windows in another order next to other windows, and as one stacked [n, 6, h, w] tensor."""
    rng = random.Random(7)
    ctxs = _windows(rng, TOP)
    lats = _latents(ctxs)
    want = [_one(decoder, c, x, [T_INIT]) for c, x in zip(ctxs, lats)]
    order = list(range(TOP))
    rng.shuffle(order)
    got = _many(decoder, [ctxs[k] for k in order], torch.stack([lats[k] for k in order]), [T_INIT])
    for g, k in zip(got, order):
        assert same(g, want[k]), ctxs[k]
    got3 = _many(decoder, ctxs[2:5], lats[2:5], [T_INIT])
    assert all(same(g, w) for g, w in zip(got3, want[2:5]))


def test_shipped_512_windows_are_bit_identical(decoder):
    """The product geometry: 512^2 windows at stride 384, a padded batch of the largest program."""
    rng = random.Random(512)
    n = TOP // 2 + 1
    ctxs = _windows(rng, n)
    lats = _latents(ctxs, 512, device="cuda")
    try:
        got = _many(decoder, ctxs, lats, [T_INIT], 512)
        for k, (ctx, lat) in enumerate(zip(ctxs, lats)):
            assert same(got[k], _one(decoder, ctx, lat, [T_INIT], 512)), (k, ctx)
    finally:
        _solve_cache(decoder).clear()         # the 512^2 programs hold gigabytes of activations
        torch.cuda.empty_cache()


def test_noise_is_the_one_window_noise(decoder, monkeypatch):
    """The noise plane a window gets inside a batch is gaussian_noise_patch at its own origin (i, j) * stride."""
    drawn = []
    real = stages.gaussian_noise_patches

    def spy(*a, **k):
        drawn.append(real(*a, **k))
        return drawn[-1]

    monkeypatch.setattr(stages, "gaussian_noise_patches", spy)
    ctxs = [(0, 5, -3), (0, -3, 5), (0, 0, 1)]
    _many(decoder, ctxs, _latents(ctxs), TWO_STEPS)
    assert len(drawn) == 2 and drawn[0].shape == (4, 1, TILE, TILE)
    for k, (_, i, j) in enumerate(ctxs):
        for step in range(2):
            want = gaussian_noise_patch(SEED + 5819 + step, i * STRIDE, j * STRIDE, TILE, TILE, 1, TILE, TILE,
                                        device="cuda")
            assert same(drawn[step][k], want), (k, step)
    swapped = gaussian_noise_patch(SEED + 5819, -3 * STRIDE, 5 * STRIDE, TILE, TILE, 1, TILE, TILE, device="cuda")
    assert not torch.equal(drawn[0][0], swapped)
    assert same(drawn[0][3], drawn[0][0])             # the padding repeats window 0


def test_nan_latent_window_gives_the_same_bits_batched_and_alone(decoder):
    ctxs = [(0, 1, 2), (0, -4, 7), (0, 3, -1)]
    lats = _latents(ctxs)
    lats[1][0, 3, 4] = float("nan")
    lats[1][5, 9, 1] = float("nan")
    lats[2][2, 0, 0] = float("inf")
    for steps in ([T_INIT], TWO_STEPS):
        got = _many(decoder, ctxs, lats, steps)
        assert torch.isnan(got[1]).any()
        for k, (ctx, lat) in enumerate(zip(ctxs, lats)):
            assert torch.equal(bits(got[k]), bits(_one(decoder, ctx, lat, steps))), (k, len(steps))


# ------------------------------------------------------------------------------------------------ the pipeline
def _cond_fn(i1, i2, j1, j2):
    gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0xFFFFFFFF)
    return torch.randn(5, i2 - i1, j2 - j1, generator=gg)


@pytest.fixture(scope="module")
def models(decoder):
    return build(COARSE_CFG).cuda(), build(BASE_CFG).cuda(), decoder


def _world(models, batch, **kw):
    coarse, base, dec = models
    return WorldPipeline.from_local_models(coarse, base, dec, seed=11, decoder_batch_size=batch, coarse_batch_size=16,
                                           decoder_tile_size=TILE, decoder_tile_stride=STRIDE, residual_mean=0.1,
                                           residual_std=1.2, conditioning_fn=_cond_fn, **kw).to("cuda").bind()


def _reads(world, order):
    """The read-outs of a world in one of two request orders."""
    reqs = {
        "residual": lambda: world.residual[:, -200:150, 40:400],
        "get": lambda: world.get(-40, -100, 200, 160, with_climate=True),
        "get_no_climate": lambda: world.get(300, -500, 420, -260, with_climate=False),
        "terrain": lambda: world.get_terrain(10, 20, 110, 150, scale=2),
    }
    names = list(reqs) if order == 0 else list(reversed(reqs))
    return {k: reqs[k]() for k in names}


def _assert_reads_equal(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, dict):
            assert x.keys() == y.keys(), (what, k)
            for q in x:
                assert (x[q] is None and y[q] is None) or same(x[q], y[q]), (what, k, q)
        else:
            assert same(x, y), (what, k)


@pytest.mark.parametrize("order", [0, 1])
def test_world_with_batched_decoder_stage_is_bit_identical(models, monkeypatch, order):
    """The latent stage solves its windows in padded batches whose programs are not batch-invariant, so what any world
    reads depends on which latent windows earlier requests computed together.  The residual canvas asks the latent
    canvas for the same windows whatever decoder_batch_size is, so worlds that see the same requests differ only in
    how the decoder batches its windows."""
    calls = []
    real = pipeline.decoder_stage_tiles

    def spy(model, seed, ctxs, *a, **k):
        calls.append(len(ctxs))
        return real(model, seed, ctxs, *a, **k)

    monkeypatch.setattr(pipeline, "decoder_stage_tiles", spy)
    ref = _world(models, 1)
    cold = _reads(ref, order)
    ref.empty_cache()
    again = _reads(ref, 1 - order)
    assert calls == [] and ref._residual.batch_size is None
    assert cold["get"]["climate"] is not None and cold["get_no_climate"]["climate"] is None
    for batch in DECODER_BATCH_SIZES[-2:]:
        calls.clear()
        world = _world(models, batch)
        _assert_reads_equal(_reads(world, order), cold, (batch, order, "cold"))
        assert 1 < max(calls) <= batch, calls
        world.empty_cache()
        _assert_reads_equal(_reads(world, 1 - order), again, (batch, order, "after empty_cache"))
        assert world._residual.batch_size == batch


def test_prebuilt_programs_cover_the_batched_decoder_solves(models, monkeypatch):
    coarse, base, dec = models
    _solve_cache(dec).clear()
    world = _world(models, TOP, torch_compile=True)
    keys = list(_solve_cache(dec))
    invariant = {k[1] for k in keys if k[-1] == "batch_invariant"}
    assert invariant == {m for m in DECODER_BATCH_SIZES if m > 1}
    assert all(len(k) == 9 for k in keys if k[-1] != "batch_invariant")     # the one-window key is unchanged
    built = []
    real = samplers.DiffusionSolve

    def spy(model, *a, **k):
        built.append(model is dec)
        return real(model, *a, **k)

    monkeypatch.setattr(samplers, "DiffusionSolve", spy)
    world.get(-300, 200, 100, 700, with_climate=True)
    assert world._residual.windows_computed > TOP
    assert not any(built), "a decoder program was built during get()"
