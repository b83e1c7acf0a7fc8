"""The batched coarse stage on the GPU: every window of `coarse_stage_tiles` is bit-identical to `coarse_stage_tile` of
the same window, and a `WorldPipeline(coarse_batch_size=16)` to one built with 1.

- tdx_coarse_condition is bit-identical to the torch op sequence of coarse_stage_tile it replaces, and
  tdx_synthetic_maps to one tdx_synthetic_map call per window, with and without imported rasters;
- the planner gives every launch of the coarse model the same (N, ksplit) at batches 1-16 in batch-invariant mode, and
  those launches, replayed at the batch sizes the pipeline pads to, match the fp64 reference (tests/_igemm_ref.py);
- random window sets (negative and non-contiguous indices) at every batch size 1-16, every coarse_pooling and the
  pool modes, with maps from a conditioning_fn and from the device synthesis with and without imports;
- the coarse canvas, get(), get_coarse and land_tiles of a world with coarse_batch_size=16 against 1, cold and after
  empty_cache(), in two request orders.

This module also registers the fenced cases of tdx_coarse_condition and tdx_synthetic_maps with
tests/test_input_extents_gpu.py (and so with tests/test_pdl_order_gpu.py) and their fenced arguments in
tests/_fence.FENCED_ARGS, and runs the same cases behind the PDL interposer itself.  It is collected before both and
imports without a GPU, so the coverage checks of a CPU-only run see the new entry points too.
"""
from __future__ import annotations

import ctypes as C
import random

import pytest
import torch

from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import WorldPipeline
from terrain_diffusion_b200.inference.noise import gaussian_noise_patch
from terrain_diffusion_b200.inference.stages import (COARSE_BATCH_SIZES, coarse_condition, coarse_stage_tile,
                                                     coarse_stage_tiles)
from terrain_diffusion_b200.inference.synthetic_map import SyntheticMap, device_imports
from terrain_diffusion_b200.inference.tiling import linear_weight_window
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests import _igemm_ref as IR
from tests import test_input_extents_gpu as IE
from tests import test_pdl_order_gpu as PO
from tests._fence import FENCED_ARGS
from tests._synthetic_inputs import stats_mapping
from tests.test_coarse_batch_cpu import recorded
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG

pytestmark = pytest.mark.gpu

F32 = torch.float32
SEED = 20261018
POOLS = (1, 2, 4, 8, 16)
MODE_PAIRS = (("avg", "avg"), ("max", "min"), ("min", "max"))


# ------------------------------------------------------------------------------------------------ fenced inputs
FENCED_ARGS["tdx_coarse_condition"] = ("map", "cond_noise", "sample_noise", "means", "stds", "cos_t", "sin_t")
FENCED_ARGS["tdx_synthetic_maps"] = ("tables", "seeds", "frequency", "scalars", "origins", "imp_values", "imp_boxes",
                                     "imp_defaults")
NEW_CASES_FROM = len(IE.CASES)


@IE.case("tdx_coarse_condition", (1, 1), (3, 37), (2, 4096))
def _condition(env, n, plane):
    m = env.inp("map", IE._rand(80 + n, n, 5, plane, lo=-3.0, hi=3.0))
    cn = env.inp("cond_noise", IE._rand(81 + n, n, 5, plane))
    sn = env.inp("sample_noise", IE._rand(82 + n, n, 6, plane))
    means = env.inp("means", IE._rand(83, 5, lo=-1.0, hi=1.0))
    stds = env.inp("stds", IE._rand(84, 5, lo=0.5, hi=2.0))
    ct = env.inp("cos_t", IE._rand(85, 5))
    st = env.inp("sin_t", IE._rand(86, 5))
    cond = env.out("cond", (n, 5, plane))
    sample = env.out("sample", (n, 6, plane))
    IE.call("tdx_coarse_condition", cond.data_ptr(), sample.data_ptr(), m.data_ptr(), cn.data_ptr(), sn.data_ptr(),
            means.data_ptr(), stds.data_ptr(), ct.data_ptr(), st.data_ptr(), 80.0, n, plane)


@IE.case("tdx_synthetic_maps", ("finalize", 1, 1, 1), ("finalize", 3, 33, 37), ("import", 2, 33, 37),
         ("import", 16, 64, 64))
def _synthetic_maps(env, kind, n, h, w):
    mode = IE.SYN_FIN | IE.SYN_SQRT if kind == "finalize" else IE.SYN_IMP | IE.SYN_SQRT
    tables = env.inp("tables", IE._tables())
    seeds = env.inp("seeds", torch.tensor([11, 22, 33, 44, 55], dtype=torch.int32), host=True)
    freq = env.inp("frequency", torch.tensor([1.5, 3, 3, 3, 3], dtype=F32) / 256, host=True)
    scalars = env.inp("scalars", torch.tensor([0.3, 1.2, 2.0, 9.0, 7.0], dtype=F32), host=True)
    org = env.inp("origins", torch.tensor([[-5 + 40 * k, 7 - 29 * k] for k in range(n)], dtype=torch.int64), host=True)
    imp = [None, None, None, 0]
    if kind == "import":
        r0 = env.inp("imp_values[0]", IE._rand(42, h // 2 + 1, w // 2 + 1, lo=-100, hi=100))
        r3 = env.inp("imp_values[3]", IE._rand(43, h, w, lo=0, hi=50))
        ptrs = torch.tensor([r0.data_ptr(), 0, 0, r3.data_ptr(), 0], dtype=torch.int64)
        vals = env.inp("imp_values", ptrs, "index", host=True, index_values=(0, 0))
        boxes = env.inp("imp_boxes", torch.tensor([[-5, 7, h // 2 + 1, w // 2 + 1], [0, 0, 0, 0], [0, 0, 0, 0],
                                                   [30, -20, h, w], [0, 0, 0, 0]], dtype=torch.int64), host=True)
        dflt = env.inp("imp_defaults", torch.tensor([0, 0, 4.5, 0, 0], dtype=F32), host=True)
        imp = [vals.data_ptr(), boxes.data_ptr(), dflt.data_ptr(), 0b00100]
    o = env.out("out", (n, 5, h, w))
    IE.call("tdx_synthetic_maps", tables.data_ptr(), 64, seeds.data_ptr(), freq.data_ptr(), scalars.data_ptr(), n,
            org.data_ptr(), h, w, mode, *imp, o.data_ptr())


NEW_CASES = IE.CASES[NEW_CASES_FROM:]


@pytest.mark.parametrize("c", NEW_CASES, ids=[c.name for c in NEW_CASES])
def test_new_entry_points_read_only_inside_their_inputs(c):
    IE.run_case(c)


@pytest.mark.parametrize("c", NEW_CASES, ids=[c.name for c in NEW_CASES])
def test_new_entry_points_wait_for_their_predecessor(c):
    PO.run_interposed(c)


# ------------------------------------------------------------------------------------------------ helpers
def bits(t):
    return t.contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def build(cfg):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
    return m


def sched():
    return EDMDPMSolverMultistepScheduler(sigma_min=0.002, sigma_max=80, sigma_data=0.5)


@pytest.fixture(scope="module")
def coarse_model():
    return build(COARSE_CFG).cuda()


COND_SNR = torch.tensor([0.3, 0.1, 1.0, 0.1, 1.0])
T_COND = torch.atan(COND_SNR)
COND_INPUTS = [v.view(-1) for v in torch.log(torch.tan(T_COND) / 8.0)]
MEANS = [0.1, -0.4, 12.0, 3.0, 700.0, 20.0]
STDS = [1.3, 0.7, 9.0, 4.0, 600.0, 15.0]


# ------------------------------------------------------------------------------------------------ the kernels
@pytest.mark.parametrize("n", [1, 3, 16])
def test_condition_kernel_is_the_torch_op_sequence_bit_for_bit(n):
    """coarse_stage_tile's ops, window by window: normalise by the model statistics of channels 0, 2-5, add the noised
    map, scale the sample noise by sigma_0."""
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(n)
    maps = (torch.randn(n, 5, 64, 64, generator=g) * 300).to(dev)
    cn = torch.randn(n, 5, 64, 64, generator=g).to(dev)
    sn = torch.randn(n, 6, 64, 64, generator=g).to(dev)
    means = torch.tensor(MEANS, device=dev)
    stds = torch.tensor(STDS, device=dev)
    sigma0 = float(sched().sigmas[0])
    cond, sample = coarse_condition(maps, cn, sn, means, stds, T_COND, sigma0)
    sel = [0, 2, 3, 4, 5]
    tc = T_COND.to(dev).view(-1, 1, 1)
    for k in range(n):
        smap = (maps[k] - means[sel, None, None]) / stds[sel, None, None]
        want = torch.cos(tc) * smap + torch.sin(tc) * cn[k]
        assert same(cond[k], want), k
        assert same(sample[k], sn[k] * sigma0), k


def test_condition_rejects_mismatched_shapes():
    dev = torch.device("cuda")
    z5, z6 = torch.zeros(2, 5, 64, 64, device=dev), torch.zeros(2, 6, 64, 64, device=dev)
    v = torch.ones(6, device=dev)
    with pytest.raises(ValueError, match="coarse_condition"):
        coarse_condition(z5, z5, z5, v, v, T_COND, 80.0)
    with pytest.raises(ValueError, match="coarse_condition"):
        coarse_condition(z5[:1], z5, z6, v, v, T_COND, 80.0)


def _imports(dev):
    """Two rasters that cover parts of the windows, one channel with a default."""
    g = torch.Generator().manual_seed(3)
    values = {0: torch.randn(90, 70, generator=g) * 800, 3: torch.rand(40, 130, generator=g) * 3000}
    origins = {0: (-60, 10), 3: (20, -100)}
    return device_imports(values, origins, {2: 4.5}, torch.device("cuda"))


@pytest.mark.parametrize("with_imports", [False, True])
@pytest.mark.parametrize("n", [1, 5, 16, 23])
def test_synthetic_windows_equal_one_call_per_window(n, with_imports):
    smap = SyntheticMap(stats_mapping(), [1.5, 3, 3, 3, 3], seed=77, device="cuda")
    rng = random.Random(n)
    origins = [(48 * rng.randint(-9, 9), 48 * rng.randint(-9, 9)) for _ in range(n)]
    imports = _imports("cuda") if with_imports else None
    got = smap.conditioning_windows(origins, 64, imports)
    assert got.shape == (n, 5, 64, 64)
    for k, (a, b) in enumerate(origins):
        assert same(got[k], smap.conditioning(a, a + 64, b, b + 64, imports)), (k, a, b)


# ------------------------------------------------------------------------------------------------ the planner
def test_batch_invariant_plans_keep_the_one_image_shape_on_this_gpu(request):
    """(N, ksplit) of every launch of the coarse forward: the one-image plan's, at every batch size 1-16, with this
    GPU's SM count and cluster occupancy.  The shapes are written to the terminal."""
    plain = [L.igemm_launch_shape(d) for d in recorded(1, False)]
    for n in range(1, 17):
        assert [L.igemm_launch_shape(d) for d in recorded(n, True)] == plain, n
    free16 = [L.igemm_launch_shape(d) for d in recorded(16, False)]
    IR.report(request.config, [f"coarse forward, batch-invariant (N, ksplit) per launch: {plain}",
                               f"coarse forward at 16 images, free plan: {free16}"])


def _replay_cases():
    """One launch per (layer shape, epilogue) of the batch-invariant coarse forward at every padded batch size."""
    out, seen = [], set()
    for n in COARSE_BATCH_SIZES:
        for d in recorded(n, True):
            case = IR.case_from_desc(d, name=f"coarse_invariant_b{n}", seed=n)
            key = (n, tuple(case.segs), case.epi, tuple(case.outs), case.resid_pnorm, case.rms_out, case.resid_inv,
                   int(d.ksplit), case.n_item)
            if key not in seen:
                seen.add(key)
                case.name += f":{len(seen)}-ks{int(d.ksplit)}"
                out.append((case, int(d.ksplit)))
    return out


@pytest.mark.parametrize("case,ksplit", _replay_cases(), ids=lambda v: v.name if isinstance(v, IR.Case) else str(v))
def test_batch_invariant_coarse_plans_match_fp64_reference(case, ksplit):
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
def _host_maps(ctxs):
    out = []
    for _, i, j in ctxs:
        g = torch.Generator().manual_seed((i * 7919 + j) & 0xFFFFFFFF)
        out.append(torch.randn(5, 64, 64, generator=g) * 2)
    return out


def _one(model, ctx, smap, pool, elev, p5):
    return coarse_stage_tile(model, sched(), SEED, ctx, smap, T_COND, COND_INPUTS,
                             linear_weight_window(64 // pool, "cuda"), MEANS, STDS, pool_size=pool,
                             elev_pool_mode=elev, p5_pool_mode=p5)


def _many(model, ctxs, smaps, pool, elev, p5):
    return coarse_stage_tiles(model, sched(), SEED, ctxs, smaps, T_COND, COND_INPUTS,
                              linear_weight_window(64 // pool, "cuda"), MEANS, STDS, pool_size=pool,
                              elev_pool_mode=elev, p5_pool_mode=p5)


def _windows(rng, n):
    """n distinct, scattered window indices, negative ones included."""
    picked = set()
    while len(picked) < n:
        picked.add((rng.randint(-40, 40), rng.randint(-40, 40)))
    return [(0, i, j) for i, j in sorted(picked, key=lambda _: rng.random())]


def test_every_batch_size_is_bit_identical_to_one_window_solves(coarse_model):
    """Random window sets at every batch size 1-16 (2, 4, 8 and 16 unpadded, the others padded), host maps."""
    rng = random.Random(1)
    for n in range(1, 17):
        ctxs = _windows(rng, n)
        maps = _host_maps(ctxs)
        got = _many(coarse_model, ctxs, maps, 1, "avg", "avg")
        assert len(got) == n
        for k, (ctx, smap) in enumerate(zip(ctxs, maps)):
            assert same(got[k], _one(coarse_model, ctx, smap, 1, "avg", "avg")), (n, k, ctx)


@pytest.mark.parametrize("pool", POOLS)
@pytest.mark.parametrize("source", ["conditioning_fn", "synthetic", "synthetic_imports"])
def test_every_pooling_mode_and_source_is_bit_identical(coarse_model, pool, source):
    """Every coarse_pooling with the pool modes, maps from host tensors or from the device synthesis (batched, with
    and without imports), at a padded (5 -> 8) and an unpadded (16) batch; the padded batch's windows come again in
    the full one, in another order, next to other windows."""
    rng = random.Random(pool)
    ctxs = _windows(rng, 16)
    if source == "conditioning_fn":
        maps = _host_maps(ctxs)
    else:
        smap = SyntheticMap(stats_mapping(), [1.5, 3, 3, 3, 3], seed=5, device="cuda")
        imports = _imports("cuda") if source == "synthetic_imports" else None
        maps = list(smap.conditioning_windows([(i * 48, j * 48) for _, i, j in ctxs], 64, imports))
    for elev, p5 in MODE_PAIRS:
        want = [_one(coarse_model, c, m, pool, elev, p5) for c, m in zip(ctxs, maps)]
        assert want[0].shape == (7, 64 // pool, 64 // pool)
        got5 = _many(coarse_model, ctxs[3:8], maps[3:8], pool, elev, p5)
        assert all(same(g, w) for g, w in zip(got5, want[3:8])), (pool, elev, p5, "batch of 5")
        order = list(range(16))
        rng.shuffle(order)
        got16 = _many(coarse_model, [ctxs[k] for k in order], [maps[k] for k in order], pool, elev, p5)
        for g, k in zip(got16, order):
            assert same(g, want[k]), (pool, elev, p5, ctxs[k])


def test_noise_is_the_one_window_noise(coarse_model):
    """coarse_stage_tiles draws the windows' noise at their own origins (one window checked against its patch)."""
    ctx = (0, -3, 7)
    a = gaussian_noise_patch(SEED, -3 * 48, 7 * 48, 64, 64, 5, 64, 64, device="cuda")
    b = gaussian_noise_patch(SEED, 7 * 48, -3 * 48, 64, 64, 5, 64, 64, device="cuda")
    assert not torch.equal(a, b)          # the origin order matters, so a swapped (y, x) would be caught below
    maps = _host_maps([ctx, (0, 7, -3)])
    got = _many(coarse_model, [ctx, (0, 7, -3)], maps, 1, "avg", "avg")
    assert same(got[0], _one(coarse_model, ctx, maps[0], 1, "avg", "avg"))


# ------------------------------------------------------------------------------------------------ the pipeline
def _cond_fn(i1, i2, j1, j2):
    gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0xFFFFFFFF)
    return torch.randn(5, i2 - i1, j2 - j1, generator=gg)


@pytest.fixture(scope="module")
def models(coarse_model):
    return coarse_model, build(BASE_CFG).cuda(), build(ounet.DECODER_CFG).cuda()


def _world(models, batch, source, pool=1):
    coarse, base, dec = models
    kw = dict(seed=11, coarse_batch_size=batch, coarse_pooling=pool, decoder_tile_size=128, decoder_tile_stride=96,
              residual_mean=0.1, residual_std=1.2)
    if source == "conditioning_fn":
        kw["conditioning_fn"] = _cond_fn
    else:
        kw["synthetic_map_stats"] = stats_mapping()
    world = WorldPipeline.from_local_models(coarse, base, dec, **kw).to("cuda").bind()
    if source == "synthetic_imports":
        g = torch.Generator().manual_seed(9)
        world.set_custom_conditioning_import(0, (torch.randn(80, 120, generator=g) * 900).numpy(), -30, -50)
        world.set_custom_conditioning_import(4, (torch.rand(50, 50, generator=g) * 40).numpy(), 10, 10,
                                             default_value=12.0)
    return world


def _reads(world, order):
    """The read-outs of a world in one of two request orders."""
    reqs = {
        "coarse": lambda: world.coarse[:, -50:50, -50:50],
        "get": lambda: world.get(-40, -100, 24, 60, with_climate=True),
        "get_coarse": lambda: world.get_coarse(-60, 40, -30, 70),
        "land": lambda: world.land_tiles(60, 1024, 0.3),
    }
    names = list(reqs) if order == 0 else list(reversed(reqs))
    return {k: reqs[k]() for k in names}


def _assert_reads_equal(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k], b[k]
        if k == "get":
            assert same(x["elev"], y["elev"]) and same(x["climate"], y["climate"]), (what, k)
        elif k == "land":
            assert x == y, (what, k)
        else:
            assert same(x, y), (what, k)


@pytest.mark.parametrize("source", ["conditioning_fn", "synthetic", "synthetic_imports"])
def test_world_with_batched_coarse_stage_is_bit_identical(models, source):
    ref = _world(models, 1, source)
    want = _reads(ref, 0)
    for order in (0, 1):
        world = _world(models, 16, source)
        cold = _reads(world, order)
        _assert_reads_equal(cold, want, (source, order, "cold"))
        world.empty_cache()
        _assert_reads_equal(_reads(world, 1 - order), want, (source, order, "after empty_cache"))
    assert world._coarse.batch_size == 16 and ref._coarse.batch_size is None


def test_one_cold_get_reaches_the_coarse_stage_as_one_batched_request(models, monkeypatch):
    """The latent canvas prefetches the union of its coarse windows, so a cold get() asks the coarse stage once, for
    all of them."""
    from terrain_diffusion_b200.inference import pipeline
    calls = []
    real = pipeline.coarse_stage_tiles

    def spy(model, scheduler, seed, ctxs, *a, **k):
        calls.append(len(ctxs))
        return real(model, scheduler, seed, ctxs, *a, **k)

    monkeypatch.setattr(pipeline, "coarse_stage_tiles", spy)
    world = _world(models, 16, "conditioning_fn")
    world.get(0, 0, 512, 512, with_climate=False)
    assert len(calls) == 1 and calls[0] == world._coarse.windows_computed > 1, calls


def test_prebuilt_programs_cover_the_batched_coarse_solves(models):
    from terrain_diffusion_b200.inference.samplers import _solve_cache
    coarse, base, dec = models
    WorldPipeline.from_local_models(coarse, base, dec, seed=1, coarse_batch_size=8, torch_compile=True,
                                    conditioning_fn=_cond_fn, decoder_tile_size=128,
                                    decoder_tile_stride=96).to("cuda").bind()
    keys = [k for k in _solve_cache(coarse) if "batch_invariant" in k]
    assert {1, 2, 4, 8} <= {k[0] for k in keys}
