"""The batch-invariant latent stage on the GPU: every tile of `latent_stage_tiles(batch_invariant=True)` is
bit-identical to a one-tile call of itself, and a `WorldPipeline(latents_batch_invariant=True)` reads the same bits
whatever its request history.

- tdx_latent_embed against an fp64 restatement of process_latent_conditioning + EDMUnet2D._host_embedding, against the
  reference's conditioning vector (stages_golden.npz), row by row against one-row launches, and with NaN, +-inf and
  zero-weight coarse cells against the torch path;
- the anchored base-model plans: (N, ksplit) at every padded batch on this GPU for both anchors, and each distinct
  launch of the shipped anchor that differs from the free plan replayed against fp64 (tests/_igemm_ref.py);
- random tile sets (negative and scattered indices) at every n from 1 to 16, both phases, host and device coarse
  windows, each tile against its one-tile call; the same tiles in other batches; NaN coarse cells; the reference's
  latent phases (stages_golden.npz);
- worlds at T = 2 and T = 1 and at coarse / decoder batch sizes of 1 and of their maxima: one big read against the same
  area read as scattered small reads in reverse order, cold and after empty_cache(), and with a cache small enough to
  evict latent tiles mid-read against an unlimited cache;
- torch_compile=True builds every anchored latent program in bind(), and get() builds no base-model program.
"""
from __future__ import annotations

import ctypes as C
import math
import random
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import WorldPipeline, pipeline, samplers
from terrain_diffusion_b200.inference.samplers import _solve_cache
from terrain_diffusion_b200.inference.stages import (LATENT_BATCH_SIZES, _concat_scales, latent_embed_spec,
                                                     latent_embedding, latent_plan_images, latent_stage_tiles,
                                                     process_latent_conditioning)
from terrain_diffusion_b200.inference.tiling import linear_weight_window
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests import _igemm_ref as IR
from tests._stage_inputs import SEED as STAGE_SEED, stage_inputs
from tests.test_latent_invariant_cpu import PADDED, recorded
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

G = np.load(Path(__file__).resolve().parent / "golden" / "stages_golden.npz")
SEED = 20261018
TOP = LATENT_BATCH_SIZES[-1]
T_INIT = math.atan(80.0 / 0.5)
T_INTER = math.atan(0.35 / 0.5)
MEANS = torch.tensor(pipeline.COND_INPUT_MEAN)
STDS = torch.tensor(pipeline.COND_INPUT_STD)
HIST = torch.tensor([[0.3, -1.2, 0.0, 2.5, 0.7]])
U = 2.0 ** -24


def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def build(cfg):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
    return m


@pytest.fixture(scope="module")
def base():
    return build(BASE_CFG).cuda()


def _coarse(n, seed=0, device="cpu"):
    """n packed [7, 4, 4] coarse windows (6 channels x w, then w), in the units of the pipeline's statistics."""
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(n, 1, 4, 4, generator=g) + 0.3
    v = MEANS[:6].view(1, 6, 1, 1) + STDS[:6].view(1, 6, 1, 1) * torch.randn(n, 6, 4, 4, generator=g)
    return torch.cat([v * w, w], dim=1).to(device)


# ------------------------------------------------------------------------------------------------ the kernel
def _embed(model, coarse, hist=HIST, t=T_INIT, means=MEANS, stds=STDS):
    spec = latent_embed_spec(model)
    n = coarse.shape[0]
    out = torch.empty((n, spec["emb_channels"]), device="cuda")
    vec = torch.empty((n, spec["cond_dims"]), device="cuda")
    latent_embedding(model, coarse.float().cuda().contiguous(), hist, means, stds, t, out, vec)
    return out, vec


def _torch_path(model, coarse, hist=HIST, t=T_INIT, means=MEANS, stds=STDS):
    """What the default latent stage computes: process_latent_conditioning + _host_embedding, fp32 torch on the GPU."""
    c = coarse.float().cuda()
    cimg = torch.cat([c[:, :-1] / c[:, -1:], torch.ones_like(c[:, :1])], dim=1)
    vec = process_latent_conditioning(cimg, hist, means, stds, torch.tensor(0.0))
    labels = torch.full((c.shape[0],), t, dtype=torch.float64).float().cuda()
    return model._host_embedding(labels, [vec]), vec


def _fp64(model, coarse, hist=HIST, t=T_INIT, means=MEANS, stds=STDS):
    """fp64 restatement of the same, from the fp32 folded weights; also returns the bound of the fp32 kernel."""
    g = {k: v.double().cpu() for k, v in model.folded().g.items()}
    c = coarse.double()
    m, s = means.double().view(1, 7, 1, 1), stds.double().view(1, 7, 1, 1)
    cimg = torch.cat([c[:, :6] / c[:, 6:], torch.ones_like(c[:, :1])], dim=1)
    x = torch.nan_to_num((cimg - m) / s, nan=float(means[0]), posinf=3.4028234663852886e38,
                         neginf=-3.4028234663852886e38)
    n = c.shape[0]
    lvl = torch.full((n, 1), (0.0 - 0.5) * math.sqrt(12), dtype=torch.float64)
    parts = [x[:, 0].flatten(1), x[:, 1].flatten(1), x[:, 2:6, 1:3, 1:3].mean(dim=(2, 3)), x[:, 6].flatten(1),
             hist.double().reshape(1, -1).expand(n, -1), lvl]
    vec = torch.cat(parts, 1) * _concat_scales([p.shape[1] for p in parts], "cpu").double()
    y = float(np.float32(t)) * g["noise_freqs"].view(1, -1)
    pe = torch.cat([torch.sin(y), torch.cos(y)], 1) * math.sqrt(2)
    silu = lambda z: z / (1 + torch.exp(-z)) / 0.596          # noqa: E731
    spec = latent_embed_spec(model)
    a_n, a_c = pe.abs() @ g["noise_linear"].abs(), vec.abs() @ g["cond0"].abs()
    pre = (pe @ g["noise_linear"] * spec["w_noise"] + silu(vec @ g["cond0"]) * spec["w_cond"]) / spec["w_norm"]
    # fp32 error of the kernel: gamma_K sum |w| |x| of each dot product (K = noise_dims + 8, cond_dims + 8 for the
    # rounding of their inputs), through the cond mp_silu and the outer one (slope <= 1.1 / 0.596 each), twice over
    slope = 1.1 / 0.596
    bound = 2 * slope * (U * (spec["noise_dims"] + 8) * a_n + slope * U * (spec["cond_dims"] + 8) * a_c) / spec["w_norm"]
    emb = silu(pre)
    return emb, vec, bound + 8 * U * emb.abs() + 1e-7


def test_kernel_matches_fp64_restatement(base):
    c = _coarse(16, seed=1)
    emb, vec = _embed(base, c)
    want, want_vec, bound = _fp64(base, c)
    assert torch.isfinite(emb).all()
    err = (emb.double().cpu() - want).abs()
    assert (err <= bound).all(), f"worst error {float((err / bound).max()):.2f}x the bound"
    assert torch.allclose(vec.double().cpu(), want_vec, rtol=1e-5, atol=2e-6)
    got_torch, _ = _torch_path(base, c)
    assert IR.rel_rms(emb.double().cpu(), got_torch.double().cpu()) < 1e-5


def test_conditioning_vector_matches_reference_golden(base):
    inp = stage_inputs()
    _, vec = _embed(base, inp["lat_cond"][:1], inp["lat_hist"], T_INIT, inp["lat_means"], inp["lat_stds"])
    np.testing.assert_allclose(vec.cpu().numpy(), G["latent_condvec"], rtol=0, atol=2e-6)


def test_every_row_is_its_one_row_launch(base):
    c = _coarse(TOP, seed=2)
    one = [_embed(base, c[r:r + 1]) for r in range(TOP)]
    for n in range(1, TOP + 1):
        emb, vec = _embed(base, c[:n])
        for r in range(n):
            assert same(emb[r], one[r][0][0]) and same(vec[r], one[r][1][0]), (n, r)


def test_non_finite_and_zero_weight_cells_follow_the_torch_path(base):
    c = _coarse(6, seed=3)
    c[0, 0, 1, 2] = float("nan")                       # a NaN value cell
    c[1, 3, 1, 1] = float("inf")                       # +inf in the climate crop
    c[2, 1, 0, 3] = float("-inf")
    c[3, 6, 2, 2] = 0.0                                # zero weight: 0 / 0 and x / 0 in every channel of that cell
    c[4, 6, 0, 0] = float("nan")                       # NaN weight
    emb, vec = _embed(base, c)
    want, want_vec = _torch_path(base, c)
    assert torch.equal(torch.isfinite(vec), torch.isfinite(want_vec))
    assert torch.equal(torch.isfinite(emb), torch.isfinite(want))
    fin = torch.isfinite(vec) & torch.isfinite(want_vec)
    assert torch.allclose(vec[fin], want_vec[fin], rtol=1e-5, atol=2e-6)
    assert torch.isfinite(emb[5]).all()                # the untouched window


def test_bad_arguments_are_rejected(base):
    out = torch.empty((2, 768), device="cuda")
    with pytest.raises(ValueError, match="coarse must be"):
        latent_embedding(base, torch.zeros((2, 7, 4, 4)), HIST, MEANS, STDS, T_INIT, out)
    with pytest.raises(ValueError, match="out must be"):
        latent_embedding(base, torch.zeros((2, 7, 4, 4), device="cuda"), HIST, MEANS, STDS, T_INIT, out[:1])
    with pytest.raises(ValueError, match="histogram values"):
        latent_embedding(base, torch.zeros((2, 7, 4, 4), device="cuda"), HIST[:, :3], MEANS, STDS, T_INIT, out)
    dummy = torch.zeros(1, device="cuda")
    p = dummy.data_ptr()
    lib = L.lib()
    for bad in (dict(n_tail=0), dict(noise_dims=6), dict(emb=2048), dict(rows=0)):
        a = {**dict(n_tail=6, noise_dims=192, emb=768, rows=1), **bad}
        rc = lib.tdx_latent_embed(p, None, p, p, p, p, a["n_tail"], p, p, p, p, a["noise_dims"], a["emb"], 1.0, 1.0,
                                  1.0, 1.4, a["rows"], L.current_stream_ptr())
        assert rc == -1 and b"latent_embed" in lib.tdx_last_error(), bad


# ------------------------------------------------------------------------------------------------ the planner
@pytest.mark.parametrize("anchor", [1, TOP])
def test_anchored_plans_keep_the_anchor_shape_on_this_gpu(request, anchor):
    """(N, ksplit) of every launch of the base forward: the anchor's free plan at every padded batch, with this GPU's
    SM count and cluster occupancy.  The split-K and image-range launches are written to the terminal."""
    plain = [L.igemm_launch_shape(d) for d in recorded(anchor, False)]
    for n in PADDED:
        assert [L.igemm_launch_shape(d) for d in recorded(n, True, anchor)] == plain, n
    split = [(int(d.height), int(d.c_out), s) for d, s in zip(recorded(anchor, False), plain) if s[1] > 1]
    IR.report(request.config, [f"base forward at 64^2 anchored at {anchor}: {len(plain)} igemm launches, "
                               f"{len(split)} split-K (h, c_out, (N, ksplit)): {split}"])


def _replay_cases():
    """Each distinct launch (layer shape, epilogue, forced shape) of the shipped anchored base forward (anchor 16) whose
    forced (N, ksplit) differs from the free plan at some padded batch, once, at the largest such batch: the launch's
    arithmetic per output tile does not depend on the image count, and the largest batch is where a forced split-K
    launch is most likely to run over image ranges.  The launches equal to the free plan are the ones the
    product-surface replay (tests/test_igemm_plans_gpu.py) already covers."""
    out, seen = [], set()
    anchor = latent_plan_images(TOP)
    for n in sorted(PADDED, reverse=True):
        free = recorded(n, False)
        for d, f in zip(recorded(n, True, anchor), free):
            if (int(d.n_per_item), int(d.ksplit)) == L.igemm_launch_shape(f):
                continue
            case = IR.case_from_desc(d, name=f"base_anchor{anchor}_b{n}", seed=n)
            key = (tuple(case.segs), case.h, case.epi, tuple(case.outs), case.resid_pnorm, case.rms_out,
                   case.resid_inv, int(d.ksplit), case.n_item)
            if key not in seen:
                seen.add(key)
                case.name += f":{len(seen)}-ks{int(d.ksplit)}"
                out.append((case, int(d.ksplit)))
    return out


@pytest.mark.parametrize("case,ksplit", _replay_cases(), ids=lambda v: v.name if isinstance(v, IR.Case) else str(v))
def test_anchored_base_plans_match_fp64_reference(case, ksplit):
    """IR.check_case with the launch's forced split-K factor (image-range launches included)."""
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
def _tiles(ctxs, device="cpu"):
    """Per tile: its packed coarse window [7, 4, 4] and a packed previous-phase window [6, 64, 64], seeded by index;
    on the device they are non-contiguous views of larger tensors."""
    conds, prevs = [], []
    for _, i, j in ctxs:
        g = torch.Generator().manual_seed((i * 7919 + j) & 0xFFFFFFFF)
        c = _coarse(1, seed=(i * 31 + j) & 0xFFFF)[0]
        big = torch.randn(6, 67, 69, generator=g) * 0.6
        big[5] = torch.rand(67, 69, generator=g) + 0.5
        big[:5] *= big[5:]
        if device == "cpu":
            conds.append(c)
            prevs.append(big[:, 2:66, 3:67].clone())
        else:
            conds.append(torch.cat([c, c], dim=2).to(device)[:, :, 4:])
            prevs.append(big.to(device)[:, 2:66, 3:67])
    return conds, prevs


def _windows(rng, n):
    picked = set()
    while len(picked) < n:
        picked.add((rng.randint(-60, 60), rng.randint(-60, 60)))
    return [(0, i, j) for i, j in sorted(picked, key=lambda _: rng.random())]


def _stage(model, ctxs, conds, prevs, phase, top=TOP):
    t, off = (T_INIT, 5819) if phase == 1 else (T_INTER, 5820)
    return latent_stage_tiles(model, SEED, ctxs, None if phase == 1 else prevs, conds, t, linear_weight_window(64, "cuda"),
                              HIST, MEANS, STDS, seed_offset=off, pad_batch_to=top, batch_invariant=True)


_ONE: dict = {}


def _one(model, ctx, cond, prev, phase):
    key = (ctx, phase)
    if key not in _ONE:
        _ONE[key] = _stage(model, [ctx], [cond.cpu()], [prev.cpu()], phase)[0].clone()
    return _ONE[key]


@pytest.mark.parametrize("device", ["cpu", "cuda"])
@pytest.mark.parametrize("phase", [1, 2])
def test_every_batch_size_is_bit_identical_to_one_tile_calls(base, phase, device):
    rng = random.Random(phase * 10 + (device == "cuda"))
    for n in range(1, TOP + 1):
        ctxs = _windows(rng, n)
        conds, prevs = _tiles(ctxs, device)
        got = _stage(base, ctxs, conds, prevs, phase)
        assert len(got) == n and got[0].shape == (6, 64, 64)
        for k, ctx in enumerate(ctxs):
            assert same(got[k], _one(base, ctx, conds[k], prevs[k], phase)), (n, k, ctx)


def test_a_tile_keeps_its_bits_in_any_batch(base):
    rng = random.Random(7)
    ctxs = _windows(rng, TOP)
    conds, prevs = _tiles(ctxs)
    for phase in (1, 2):
        want = [_one(base, c, x, p, phase) for c, x, p in zip(ctxs, conds, prevs)]
        for trial in range(4):
            order = rng.sample(range(TOP), rng.randint(2, TOP))
            got = _stage(base, [ctxs[k] for k in order], [conds[k] for k in order], [prevs[k] for k in order], phase)
            assert all(same(g, want[k]) for g, k in zip(got, order)), (phase, trial)


def test_nan_coarse_cells_give_the_same_bits_batched_and_alone(base):
    ctxs = [(0, 1, 2), (0, -4, 7), (0, 3, -1), (0, 9, 9), (0, -2, -8)]
    conds, prevs = _tiles(ctxs)
    conds[1][0, 1, 1] = float("nan")
    conds[2][3, 2, 2] = float("nan")
    conds[3][6, 0, 0] = 0.0
    for phase in (1, 2):
        got = _stage(base, ctxs, conds, prevs, phase)
        for k, ctx in enumerate(ctxs):
            assert same(got[k], _stage(base, [ctx], [conds[k]], [prevs[k]], phase)[0]), (phase, k)


def test_invariant_stage_matches_reference_method(base):
    """The latent phases of stages_golden.npz (reference method bodies) at the tolerance of tests/test_stages_gpu.py;
    the weight plane bit-exact."""
    inp = stage_inputs()
    ww = linear_weight_window(64)
    sig0 = float(EDMDPMSolverMultistepScheduler().sigmas[0])
    ctxs = [(0, 1, 2), (0, -1, 0)]

    def check(got, want):
        got, want = got.cpu(), torch.from_numpy(want)
        assert torch.equal(got[-1], want[-1])
        assert IR.rel_rms(got[:-1].double(), want[:-1].double()) < 1e-2

    p1 = latent_stage_tiles(base, STAGE_SEED, ctxs, None, [c.clone() for c in inp["lat_cond"]], math.atan(sig0 / 0.5),
                            ww, inp["lat_hist"], inp["lat_means"], inp["lat_stds"],
                            seed_offset=int(G["latent_seed_offsets"][0]), pad_batch_to=16, batch_invariant=True)
    for got, want in zip(p1, G["latent_phase1"]):
        check(got, want)
    prev = [torch.from_numpy(x) for x in G["latent_phase1"]]
    p2 = latent_stage_tiles(base, STAGE_SEED, ctxs, prev, [c.clone() for c in inp["lat_cond"]], math.atan(0.35 / 0.5),
                            ww, inp["lat_hist"], inp["lat_means"], inp["lat_stds"],
                            seed_offset=int(G["latent_seed_offsets"][1]), batch_invariant=True)
    for got, want in zip(p2, G["latent_phase2"]):
        check(got, want)


# ------------------------------------------------------------------------------------------------ the pipeline
DTILE, DSTRIDE = 128, 96


def _cond_fn(i1, i2, j1, j2):
    gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0xFFFFFFFF)
    return torch.randn(5, i2 - i1, j2 - j1, generator=gg)


@pytest.fixture(scope="module")
def models(base):
    return build(COARSE_CFG).cuda(), base, build(ounet.DECODER_CFG).cuda()


def _world(models, T, cb, db, **kw):
    coarse, base_m, dec = models
    return WorldPipeline.from_local_models(coarse, base_m, dec, seed=11, T=T, latents_batch_invariant=True,
                                           coarse_batch_size=cb, decoder_batch_size=db, decoder_tile_size=DTILE,
                                           decoder_tile_stride=DSTRIDE, residual_mean=0.1, residual_std=1.2,
                                           conditioning_fn=_cond_fn, **kw).to("cuda").bind()


LAT = (-40, 40, -20, 76)                    # latent rows / columns read in one piece and in pieces
GET = (-200, -120, 200, 250)                # get() area in pixels


def _big(world, order=0):
    a, b, c, d = LAT
    i1, j1, i2, j2 = GET
    reqs = {
        "latents": lambda: world.latents[:, a:b, c:d],
        "residual": lambda: world.residual[:, i1:i2, j1:j2],
        "get": lambda: world.get(i1, j1, i2, j2, with_climate=True),
        "get_no_climate": lambda: world.get(i1 + 40, j1, i2, j2 - 30, with_climate=False),
        "terrain": lambda: world.get_terrain(i1 // 2, j1 // 2, i2 // 2, j2 // 2, scale=2),
    }
    names = list(reqs) if order == 0 else list(reversed(reqs))
    return {k: reqs[k]() for k in names}


def _small_latents(world):
    """LAT read as 20 x 24 blocks, scattered, in reverse row-major order, assembled on the host."""
    a, b, c, d = LAT
    out = torch.empty((6, b - a, d - c))
    blocks = [(y, x) for y in range(a, b, 20) for x in range(c, d, 24)]
    for y, x in reversed(blocks):
        y2, x2 = min(y + 20, b), min(x + 24, d)
        out[:, y - a:y2 - a, x - c:x2 - c] = world.latents[:, y:y2, x:x2]
    return out


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


_REFERENCE: dict = {}


@pytest.mark.parametrize("T", [2, 1])
@pytest.mark.parametrize("cb,db", [(1, 1), (16, 4)])
def test_world_reads_do_not_depend_on_request_history(models, monkeypatch, T, cb, db):
    sizes = []
    real = pipeline.latent_stage_tiles

    def spy(model, seed, ctxs, *a, **k):
        assert k.get("batch_invariant") is True
        sizes.append(len(ctxs))
        return real(model, seed, ctxs, *a, **k)

    monkeypatch.setattr(pipeline, "latent_stage_tiles", spy)
    if T not in _REFERENCE:       # one cold big read per T: the batch sizes do not change a world's bits
        _REFERENCE[T] = _big(_world(models, T, 16, 4, cache_limit=None))
    want = _REFERENCE[T]
    assert want["get"]["climate"] is not None and want["get_no_climate"]["climate"] is None
    # the same area as scattered small reads in reverse order, then the big reads on that warm cache
    world = _world(models, T, cb, db, cache_limit=None)
    assert same(_small_latents(world), want["latents"])
    _assert_reads_equal(_big(world, 1), want, (T, cb, db, "after small reads"))
    world.empty_cache()
    _assert_reads_equal(_big(world, 1), want, (T, cb, db, "after empty_cache"))
    # a cache of 24 latent tiles per canvas: latent tiles are evicted and solved again mid-read, in other batches
    tight = _world(models, T, cb, db, cache_limit=24 * 6 * 64 * 64 * 4)
    assert same(_small_latents(tight), want["latents"])
    _assert_reads_equal(_big(tight), want, (T, cb, db, "evicting cache"))
    assert tight._latents.windows_evicted > 0
    assert len(set(sizes)) >= 3 and max(sizes) > 1, sorted(set(sizes))


def test_prebuilt_programs_cover_the_anchored_latent_solves(models, monkeypatch):
    coarse, base_m, dec = models
    _solve_cache(base_m).clear()
    world = _world(models, 2, 16, 4, torch_compile=True)
    keys = [k for k in _solve_cache(base_m) if k[0] == "cm"]
    assert {k[1] for k in keys} == set(PADDED)
    anchor = latent_plan_images(TOP)
    suffix = ("batch_invariant",) if anchor == 1 else ("plan_images", anchor, "batch_invariant")
    assert all(k[-len(suffix):] == suffix for k in keys)
    assert len(keys) == 2 * len(PADDED)                 # both phases
    built = []
    real = samplers.DiffusionSolve

    def spy(model, *a, **k):
        built.append(model is base_m)
        return real(model, *a, **k)

    monkeypatch.setattr(samplers, "DiffusionSolve", spy)
    world.get(-300, 200, 100, 700, with_climate=True)
    assert world._latents.windows_computed > TOP
    assert not any(built), "a base-model program was built during get()"
