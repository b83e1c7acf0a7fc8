"""The launch program (csrc/tdx_program.cu) against its own launches run one at a time.

A program replays a recorded launch list as one CUDA graph whose kernels overlap through programmatic dependent launch
(PDL): each kernel may start before the previous one ends and must wait (griddepcontrol.wait) before it touches what
an earlier launch writes or reads.  No kernel behind a program uses atomics outside the debug hooks, and split-K and
the cluster pixel-norm exchange partial results through fixed slots, so a program's results do not depend on how its
launches are issued: every way of issuing one is compared BIT FOR BIT with the serialized replay, in which every
recorded descriptor goes through its own public entry point (tdx_igemm_run, tdx_im2col_run, tdx_conv_out_run,
tdx_embed_run, tdx_attn_run) with a device synchronise after each.  The modes:

  graph      tdx_program_run(use_graph=1), the shipped path, twice from the same state
  eager      tdx_program_run(use_graph=0)
  profile    tdx_program_profile (also: one finite time and the fixed kind code per launch)
  capture    tdx_program_run(use_graph=1) issued inside a caller's torch.cuda.CUDAGraph capture, then replayed
  side       graph replay on a torch side stream whose inputs torch wrote on that stream just before

Every mode starts from the same state: each buffer the program writes filled with NaN, every other buffer (inputs,
and the sample / x0_prev a solve updates in place) restored from a snapshot.  The whole state is compared -- every
activation, pixel-norm plane, modulation vector and the solver buffers -- so a difference names the buffer, and the
launch that wrote it.  Each mode runs once.

Besides the shipped programs, a hand-built chain puts the hazards PDL must respect next to each other on tiny
launches, and each of its launches is checked against fp64 from the inputs it actually read (tests/_igemm_ref.py and
the restatements of test_direct_kernels_gpu.py), so the chain is a correct computation and not only a reproducible
one.  The last part checks the program API's contract: what `add` copies, when the graph is captured again, failed
adds, new values in the same buffers, streams, the empty program and a second device.
"""
from __future__ import annotations

import ctypes as C
import gc
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import autoencoder as oae
from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import DiffusionSolve
from terrain_diffusion_b200.inference.solve import consistency_rows
from terrain_diffusion_b200.layout import from_nc8hw8, pack_weight_segments, to_nc8hw8
from terrain_diffusion_b200.models import EDMAutoencoder, EDMUnet2D
from terrain_diffusion_b200.models.plan import UNetProgram
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests._capture import CONFIGS
from tests._igemm_ref import (case_from_desc, elementwise_ratio, needs_norm, plan_of, reference, rel_rms,
                              report)
from tests.test_direct_kernels_gpu import _conv_out_weight_layout, _sched_update_fp32

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
KIND_CODE = {"igemm": 1, "conv_out": 2, "embed": 3, "attn": 4, "im2col": 5}
"""The launch kinds tdx_program_profile reports (fixed codes: bench.py selects igemm = 1)."""
KERNEL_KIND = {"igemm_kernel": "igemm", "conv_out_kernel": "conv_out", "embed_kernel": "embed",
               "attn_kernel": "attn", "im2col_in_kernel": "im2col"}


@pytest.fixture(scope="module")
def summary(request):
    """Programs and modes compared, and the worst fp64 share of the hazard chain; written to the terminal (also
    under -q) when the module is done."""
    found = {"compared": [], "share": {}}
    yield found
    lines = [f"program {name}: {n} launches, bit-identical to the serialized replay in modes {', '.join(modes)}"
             for name, n, modes in found["compared"]]
    lines += [f"hazard chain: worst {kind}: {v[0]:.3f} ({v[1]})" for kind, v in sorted(found["share"].items())]
    report(request.config, lines)


def _note(summary, kind, value, where):
    if kind not in summary["share"] or value > summary["share"][kind][0]:
        summary["share"][kind] = (value, where)


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ------------------------------------------------------------------------------------------------ program state
def _written(kind, d):
    """(pointers launch `d` only writes, pointers it reads and writes in place)."""
    if kind == "igemm":
        return [o.ptr for o in d.out if o.kind != L.OUT_NONE] + ([d.rms_out] if d.rms_out else []), []
    if kind in ("im2col", "attn"):
        return [d.out], []
    if kind == "embed":
        return [d.blocks[i].cvec for i in range(d.n_blocks)], []
    inout = [d.sample, d.x0_prev] if d.sched_coef else []
    return ([d.model_out] if d.model_out else []), inout


class Subject:
    """One program under test: its handle, its recorded launches [(kind, descriptor copy, original descriptor)] and
    its state {name: device tensor}.  `start` is the state every mode starts from: NaN in what the launches write,
    except in the buffers they update in place and in `inputs` (read before a later launch overwrites them)."""

    def __init__(self, name, prog, launches, state, device=DEV, inputs=()):
        self.name, self.prog, self.launches, self.state, self.device = name, prog, launches, state, device
        by_ptr = {t.data_ptr(): k for k, t in state.items()}
        self.writer = {}                # buffer name -> index of the first launch that writes it
        nan, inout = set(), set()
        for i, (kind, d, _) in enumerate(launches):
            w, io = _written(kind, d)
            for p in w + io:
                assert p in by_ptr, f"{name}: launch {i} ({kind}) writes a buffer outside the recorded state"
                self.writer.setdefault(by_ptr[p], i)
            nan |= {by_ptr[p] for p in w}
            inout |= {by_ptr[p] for p in io}
        self.nan = nan - inout - set(inputs)
        self.start = {}
        for k, t in state.items():
            self.start[k] = torch.full_like(t, float("nan")) if k in self.nan else t.clone()

    @property
    def handle(self):
        return self.prog.handle

    def reset(self):
        for k, t in self.state.items():
            t.copy_(self.start[k])

    def snapshot(self):
        return {k: t.clone() for k, t in self.state.items()}

    def order(self, names):
        return sorted(names, key=lambda k: (self.writer.get(k, -1), k))


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def assert_identical(sub, got, want, mode):
    bad = sub.order([k for k in want if not _same_bits(got[k], want[k])])
    if bad:
        first = bad[0]
        i = sub.writer.get(first)
        where = f"launch {i} ({sub.launches[i][0]})" if i is not None else "no launch"
        raise AssertionError(f"{sub.name}, mode {mode}: {len(bad)} of {len(want)} buffers differ from the serialized "
                             f"replay; first {first!r}, written by {where}; all: {bad[:12]}")


# ------------------------------------------------------------------------------------------------ the modes
def _run_one(kind, d, device):
    with torch.cuda.device(device):
        L.check(getattr(L.lib(), f"tdx_{kind}_run")(C.byref(d), L.current_stream_ptr(device)))
        torch.cuda.synchronize(device)


def serialized(sub, trace=None):
    """(a) every recorded descriptor through its own entry point, synchronised after each.  trace: list that gets the
    state before every launch (and, last, the final state)."""
    for kind, d, _ in sub.launches:
        if trace is not None:
            trace.append(sub.snapshot())
        _run_one(kind, d, sub.device)
    if trace is not None:
        trace.append(sub.snapshot())


def mode_graph(sub):
    L.call(L.lib().tdx_program_run, sub.device, sub.handle, 1)


def mode_eager(sub):
    L.call(L.lib().tdx_program_run, sub.device, sub.handle, 0)


def mode_profile(sub):
    n = L.lib().tdx_program_num_launches(sub.handle)
    assert n == len(sub.launches), (n, len(sub.launches))
    ms = (C.c_float * max(n, 1))(*([-1.0] * max(n, 1)))
    kinds = (C.c_int32 * max(n, 1))()
    L.call(L.lib().tdx_program_profile, sub.device, sub.handle, ms, kinds)
    times = list(ms)[:n]
    assert all(math.isfinite(t) and t >= 0.0 for t in times), times
    assert list(kinds)[:n] == [KIND_CODE[k] for k, _, _ in sub.launches]


def mode_capture(sub):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        L.call(L.lib().tdx_program_run, sub.device, sub.handle, 1)
    sub.reset()
    g.replay()
    torch.cuda.synchronize()
    del g


def mode_side(sub):
    main = torch.cuda.current_stream(sub.device)
    side = torch.cuda.Stream(sub.device)
    side.wait_stream(main)
    with torch.cuda.stream(side):
        sub.reset()                   # the inputs, written by torch on the side stream just before the replay
        L.call(L.lib().tdx_program_run, sub.device, sub.handle, 1)
    main.wait_stream(side)


MODES = [("graph", mode_graph), ("graph again", mode_graph), ("eager", mode_eager), ("profile", mode_profile),
         ("capture", mode_capture), ("side", mode_side)]


def compare_modes(sub, want):
    for name, run in MODES:
        sub.reset()
        torch.cuda.synchronize()
        run(sub)
        torch.cuda.synchronize()
        assert_identical(sub, sub.snapshot(), want, name)
    return [m for m, _ in MODES]


def serialized_reference(sub):
    """The state the serialized replay leaves, after checking that it writes every buffer it is meant to write."""
    sub.reset()
    serialized(sub)
    want = sub.snapshot()
    unwritten = sub.order([k for k in sub.nan if torch.isnan(want[k].float()).any()])
    assert not unwritten, f"{sub.name}: buffers the serialized replay leaves (partly) unwritten: {unwritten}"
    return want


# ------------------------------------------------------------------------------------------------ shipped programs
def _recording(monkeypatch):
    """Wrap UNetProgram.add: [(kind, descriptor copy, original descriptor)].  The original is kept alive because the
    copy of an embed descriptor points into the block array the original owns (plan.py does not keep it)."""
    launches = []
    add = UNetProgram.add

    def recording_add(self, kind, desc):
        launches.append((kind, type(desc).from_buffer_copy(desc), desc))
        add(self, kind, desc)
    monkeypatch.setattr(UNetProgram, "add", recording_add)
    return launches


def _collect(obj, path, found):
    if isinstance(obj, torch.Tensor):
        if obj.is_cuda and obj.numel():
            p = obj.data_ptr()
            if p not in found or obj.numel() > found[p][1].numel():       # of views at one address, keep the largest
                found[p] = (path, obj)
    elif isinstance(obj, dict):
        for k, v in obj.items():
            _collect(v, f"{path}{k}" if not path else f"{path}.{k}", found)
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            _collect(v, f"{path}[{i}]", found)


def program_state(prog, named=()):
    """Every device tensor a UNetProgram keeps alive (activation arenas, pixel-norm planes, modulation vectors,
    inputs, solver buffers), named by where it is kept; `named` [(name, tensor)] overrides the name."""
    found = {}
    tags = {id(prog.arena): "", id(prog.cvecs): "cvec "}     # other dicts (a guide's arena, sched) get "d<i>:"
    for i, item in enumerate(prog.keep):
        for j, part in enumerate(item if isinstance(item, tuple) else (item,)):
            if isinstance(part, dict):
                tag = tags.setdefault(id(part), f"d{len(tags) - 2}:")
                for k, t in part.items():
                    _collect(t, tag + str(k), found)
            else:
                _collect(part, f"keep[{i}][{j}]", found)
    for name, t in named:
        found[t.data_ptr()] = (name, t)
    return {name: t for name, t in found.values()}


def _model(cfg, seed=0):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(ounet.procedural_state_dict(cfg, seed=seed))
    return m.to(DEV)


def _cond(cfg, n, g):
    return [(torch.randn(n, dim, generator=g) if kind == "tensor" else torch.randn(n, generator=g)).to(DEV)
            for kind, dim, _ in cfg.get("conditional_inputs") or []]


def build_subject(name, monkeypatch):
    """Run one public call with the launch recording on; return its program as a Subject."""
    launches = _recording(monkeypatch)
    g = torch.Generator().manual_seed(11)
    named = []
    if name in ("decoder", "base", "coarse"):
        cfg = CONFIGS[name]
        n, h, w = {"decoder": (2, 64, 128), "base": (1, 64, 128), "coarse": (2, 16, 24)}[name]
        m = _model(cfg)
        x = torch.randn(n, cfg["in_channels"], h, w, generator=g).to(DEV)
        m(x, torch.tensor([0.4, 1.1][:n], device=DEV), _cond(cfg, n, g))
        prog = next(iter(m._plans.values()))[0]
        owner = m
    elif name in ("decoder solve", "guided solve"):
        cfg = CONFIGS["decoder"]
        m = _model(cfg)
        guide = _model(cfg, seed=1) if name == "guided solve" else None
        n, steps = 2, (3 if guide is None else 2)
        solve = DiffusionSolve(m, EDMDPMSolverMultistepScheduler(), n, 64, 128, steps, guide=guide,
                               guidance_scale=1.5 if guide is not None else 1.0)
        solve.run((torch.randn(n, 1, 64, 128, generator=g) * 80).to(DEV), torch.randn(n, 4, 64, 128, generator=g).to(DEV))
        prog = solve.prog
        named = [("sample", solve.sample), ("x0_prev", solve.x0_prev)]
        if guide is not None:
            named.append(("guide_out", solve.guide_out))
        owner = (m, guide, solve)
    elif name == "consistency solve":
        cfg = CONFIGS["base"]
        m = _model(cfg)
        n = 2
        solve = DiffusionSolve(m, None, n, 64, 128, 1, coef_rows=consistency_rows(1.2, from_unit_noise=True))
        solve.run(torch.randn(n, cfg["out_channels"], 64, 128, generator=g).to(DEV), None,
                  conditional_inputs=_cond(cfg, n, g))
        prog = solve.prog
        named = [("sample", solve.sample), ("x0_prev", solve.x0_prev)]
        owner = (m, solve)
    elif name in ("autoencoder preencode", "autoencoder decode"):
        ae = EDMAutoencoder(**oae.X8_CFG).eval()
        ae.load_state_dict(oae.procedural_state_dict(oae.X8_CFG, seed=0))
        ae = ae.to(DEV)
        if name == "autoencoder preencode":
            ae.preencode(torch.randn(1, 1, 64, 128, generator=g).to(DEV))
            prog = next(iter(ae.encoder._plans.values()))[0]
        else:
            ae.decode(torch.randn(2, 4, 8, 16, generator=g).to(DEV))
            prog = next(iter(ae._plans.values()))[0]
        owner = ae
    else:
        raise KeyError(name)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert len(launches) == prog.n_launch == L.lib().tdx_program_num_launches(prog.handle)
    sub = Subject(name, prog, launches, program_state(prog, named))
    sub.owner = owner
    return sub


PROGRAMS = ["decoder", "base", "coarse", "decoder solve", "guided solve", "consistency solve",
            "autoencoder preencode", "autoencoder decode"]


@pytest.mark.parametrize("name", PROGRAMS)
def test_shipped_program_is_bit_identical_however_it_is_issued(name, monkeypatch, summary):
    sub = build_subject(name, monkeypatch)
    kinds = [k for k, _, _ in sub.launches]
    if name in ("base", "consistency solve"):
        assert "attn" in kinds, name
    want = serialized_reference(sub)
    modes = compare_modes(sub, want)
    summary["compared"].append((name, len(sub.launches), modes))


def test_shipped_programs_plan_split_k_and_pixel_norm_clusters(monkeypatch):
    """The programs above include at least one split-K launch and one launch whose pixel-norm statistics travel
    through a cluster (the two paths that exchange partial results between CTAs)."""
    seen = set()
    for name in ("base", "decoder solve"):
        sub = build_subject(name, monkeypatch)
        for kind, d, _ in sub.launches:
            if kind != "igemm":
                continue
            case = case_from_desc(d)
            p = plan_of(case)
            if p["ks"] > 1:
                seen.add("split-K")
            if needs_norm(case) and p["cluster"] > 1:
                seen.add("pixel-norm cluster")
        del sub
    assert seen == {"split-K", "pixel-norm cluster"}, seen


# ------------------------------------------------------------------------------------------------ hazard chain
HW = 8
"""The chain runs on one 8 x 8 image: every launch is a handful of CTAs, so the overlap PDL allows is proportionally
largest."""


def _nc8(c, g, device, scale=1.0):
    return to_nc8hw8(torch.randn(1, c, HW, HW, generator=g, device=device) * scale)


class Chain:
    """A program written out by hand, on its own buffers, with the hazards PDL must respect next to each other:

      0  embed    emb_a -> cvec                              modulation vectors
      1  igemm    x -> h1 (3x3, 768 ch, EMB_SILU with cvec)   split-K
      2  igemm    h1 -> h2 (3x3, 768 ch)                     split-K: shares the per-device scratch with launch 1
      3  igemm    h2 -> x (1x1) + rms_out inv                pixel-norm cluster; overwrites launch 1's input
      4  igemm    h2 -> q (1x1)
      5  igemm    h2 -> z (1x1) + 0.7 pixelnorm(x) via inv    reads x and inv, written two launches back
      6  attn     (q, z, x) -> h1                            overwrites what launches 2 and 4 read
      7  igemm    h1 -> d (1x1, 768 -> 128)
      8  conv_out d -> model_out; sample, x0_prev updated in place
      9  im2col   sample * c_in -> cols                      reads the sample launch 8 just updated
     10  embed    emb_b -> cvec                              rewrites the rows launch 1 read
     11  igemm    cols -> y (1x1, 64 -> 768, EMB_SILU with the new cvec)
    """

    C = 768

    def __init__(self, seed, device=DEV):
        self.device = device
        g = torch.Generator(device=device).manual_seed(seed)
        c = self.C
        st = {}
        st["x"] = _nc8(c, g, device)
        for k in ("h1", "h2", "q", "z", "y"):
            st[k] = torch.empty_like(st["x"])
        st["d"] = torch.empty((1, 128 // 8, HW, HW, 8), dtype=torch.bfloat16, device=device)
        st["cols"] = torch.empty((1, 64 // 8, HW, HW, 8), dtype=torch.bfloat16, device=device)
        st["inv"] = torch.empty((1, HW, HW), dtype=torch.float32, device=device)
        st["cvec"] = torch.empty((1, c), dtype=torch.float32, device=device)
        st["emb_a"] = torch.randn(1, c, generator=g, device=device)
        st["emb_b"] = torch.randn(1, c, generator=g, device=device)
        st["model_out"] = torch.empty((1, 5, HW, HW), dtype=torch.float32, device=device)
        st["sample"] = torch.randn(1, 5, HW, HW, generator=g, device=device) * 3
        st["x0_prev"] = torch.randn(1, 5, HW, HW, generator=g, device=device)
        st["coef"] = torch.tensor([0.9173, 0.4121, 0.3377, -0.2719], dtype=torch.float32, device=device)
        st["c_in"] = torch.tensor([0.37], dtype=torch.float32, device=device)
        self.state = st
        self.keep = []
        self.arrays = []
        self.checks = []
        self.launches = []
        self.start = None

        def w(cout, cin, k):
            return (torch.randn(cout, cin, k, k, generator=g, device=device) / (cin * k * k) ** 0.5).bfloat16().float()

        self.w_emb = (torch.randn(c, c, generator=g, device=device) * (0.8 / c ** 0.5)).contiguous()
        self._embed("emb_a")
        self._igemm([("x", 9)], w(c, c, 3), ["h1"], epi=L.EPI_EMB_SILU)
        self._igemm([("h1", 9)], w(c, c, 3), ["h2"])
        self._igemm([("h2", 1)], w(c, c, 1), ["x"], rms="inv")
        self._igemm([("h2", 1)], w(c, c, 1), ["q"])
        self._igemm([("h2", 1)], w(c, c, 1), ["z"], resid="x", resid_inv="inv")
        self._attn("q", "z", "x", "h1")
        self._igemm([("h1", 1)], w(128, c, 1), ["d"])
        self.w_out = torch.randn(5, 128, 3, 3, generator=g, device=device) / (9 * 128) ** 0.5
        self._conv_out()
        self._im2col()
        self._embed("emb_b")
        self._igemm([("cols", 1)], w(c, 64, 1), ["y"], epi=L.EPI_EMB_SILU)

    def _add(self, kind, d, check):
        self.launches.append((kind, d, d))
        self.checks.append(check)

    def _embed(self, src):
        st = self.state
        arr = (L.TdxEmbedBlock * 1)()
        arr[0].weight, arr[0].cvec, arr[0].c_out = self.w_emb.data_ptr(), st["cvec"].data_ptr(), self.C
        d = L.TdxEmbedDesc()
        d.emb_in, d.emb_channels, d.n_img, d.n_blocks, d.blocks = st[src].data_ptr(), self.C, 1, 1, arr
        self.arrays.append(arr)

        def check(before, after, note):
            c = before[src].double() @ self.w_emb.double() + 1.0
            ref = c / (c.square().mean(dim=1, keepdim=True) + 1e-8).sqrt()
            err = float((after["cvec"].double() - ref).abs().max())
            note("embed cvec (x 2e-5 abs)", err / 2e-5)
        self._add("embed", d, check)

    def _igemm(self, segs, wt, outs, epi=0, rms=None, resid=None, resid_inv=None):
        st = self.state
        cout = wt.shape[0]
        chans = [(st[k].shape[1] * 8, taps) for k, taps in segs]
        d = L.TdxIgemmDesc()
        for i, ((k, taps), (ch, _)) in enumerate(zip(segs, chans)):
            d.a_ptr[i], d.a_channels[i], d.a_taps[i] = st[k].data_ptr(), ch, taps
        d.n_seg = len(segs)
        d.n_per_item = L.igemm_choose_n(cout, 1, HW, HW, chans)
        b = pack_weight_segments([wt], d.n_per_item).to(self.device)
        self.keep.append(b)
        d.b_packed, d.c_out = b.data_ptr(), cout
        d.n_img, d.height, d.width = 1, HW, HW
        d.epi_flags = epi | (L.EPI_RESID if resid else 0)
        if epi & L.EPI_EMB_SILU:
            d.cvec = st["cvec"].data_ptr()
        if resid:
            d.resid, d.resid_spatial, d.resid_scale = st[resid].data_ptr(), L.SP_SAME, 0.7
            d.resid_inv = st[resid_inv].data_ptr()
        if rms:
            d.rms_out = st[rms].data_ptr()
        for i, k in enumerate(outs):
            d.out[i].ptr, d.out[i].kind, d.out[i].spatial, d.out[i].scale = st[k].data_ptr(), L.OUT_RAW, L.SP_SAME, 1.0

        def check(before, after, note):
            case = case_from_desc(d, name=f"igemm -> {outs[0]}")
            acts = [from_nc8hw8(before[k]) for k, _ in segs]
            cvec = before["cvec"] if epi & L.EPI_EMB_SILU else torch.ones(1, cout, device=self.device)
            res = torch.zeros(1, cout, HW, HW, device=self.device)
            if resid:
                # the residual's pixel-norm with the 1 / (eps + rms) plane an earlier launch stored, not recomputed
                case.resid_pnorm = 0
                res = from_nc8hw8(before[resid]).double() * before[resid_inv].double()[:, None]
            refs = reference(case, acts, [wt], cvec, res)
            gots = [from_nc8hw8(after[k]) for k in outs] + ([after[rms]] if rms else [])
            for i, (got, ref) in enumerate(zip(gots, refs)):
                if i < len(outs):
                    assert rel_rms(got.double(), ref.bfloat16().double()) < 2e-3, case.name
                note("igemm (x per-element bound)", elementwise_ratio(got, ref))
        self._add("igemm", d, check)

    def _attn(self, q, k, v, out):
        st = self.state
        d = L.TdxAttnDesc()
        d.q, d.k, d.v, d.out = st[q].data_ptr(), st[k].data_ptr(), st[v].data_ptr(), st[out].data_ptr()
        heads, tokens = self.C // 64, HW * HW
        d.n_img, d.heads, d.head_dim, d.tokens = 1, heads, 64, tokens

        def check(before, after, note):
            def norm(name):
                t = from_nc8hw8(before[name]).double().reshape(1, heads, 64, tokens)
                return t / (1e-4 + t.square().mean(dim=2, keepdim=True).sqrt())
            qn, kn, vn = norm(q), norm(k), norm(v)
            wts = torch.softmax(torch.einsum("nhdq,nhdk->nhqk", qn, kn) / 8.0, dim=-1)
            ref = torch.einsum("nhqk,nhdk->nhdq", wts, vn)
            got = from_nc8hw8(after[out]).reshape(1, heads, 64, tokens)
            note("attention (x per-element bound)", elementwise_ratio(got, ref))
        self._add("attn", d, check)

    def _conv_out(self):
        st = self.state
        self.w_out_layout = _conv_out_weight_layout(self.w_out)
        d = L.TdxConvOutDesc()
        d.x, d.c_in, d.weight, d.c_out = st["d"].data_ptr(), 128, self.w_out_layout.data_ptr(), 5
        d.n_img, d.height, d.width = 1, HW, HW
        d.model_out, d.sched_coef = st["model_out"].data_ptr(), st["coef"].data_ptr()
        d.sample, d.x0_prev = st["sample"].data_ptr(), st["x0_prev"].data_ptr()

        def check(before, after, note):
            x = from_nc8hw8(before["d"]).double()
            ref = F.conv2d(x, self.w_out.double(), padding=1)
            scale = F.conv2d(x.abs(), self.w_out.double().abs(), padding=1)
            f = after["model_out"]
            note("conv_out model_out (x 2^-17 sum|terms|)", float(((f.double() - ref).abs() / (2.0 ** -17 * scale)).max()))
            want_s, want_x0 = _sched_update_fp32(before["sample"], f, before["x0_prev"], before["coef"])
            assert torch.equal(after["sample"], want_s) and torch.equal(after["x0_prev"], want_x0)
        self._add("conv_out", d, check)

    def _im2col(self):
        st = self.state
        d = L.TdxIm2colDesc()
        d.src[0], d.src_channels[0], d.src_dtype[0] = st["sample"].data_ptr(), 5, 0
        d.src_scale[0] = st["c_in"].data_ptr()
        d.out, d.k_pad, d.n_img, d.height, d.width = st["cols"].data_ptr(), 64, 1, HW, HW

        def check(before, after, note):
            x = before["sample"].double() * before["c_in"].double()
            x = torch.cat([x, torch.ones_like(x[:, :1])], dim=1)                    # [1, 6, h, w]
            cols = F.unfold(x, 3, padding=1).reshape(1, 6, 9, HW, HW).transpose(1, 2).reshape(1, 54, HW, HW)
            ref = torch.cat([cols, torch.zeros(1, 10, HW, HW, dtype=cols.dtype, device=cols.device)], dim=1)
            note("im2col (x per-element bound)", elementwise_ratio(from_nc8hw8(after["cols"]), ref))
        self._add("im2col", d, check)

    def program(self, upto=None):
        prog = UNetProgram(self.device)
        for kind, d, _ in self.launches[:upto]:
            prog.add(kind, d)
        return prog

    def subject(self, prog, name="hazard chain"):
        """Every subject of one chain starts from the state the chain was built with."""
        sub = Subject(name, prog, self.launches, self.state, self.device, inputs=("x",))
        if self.start is None:
            self.start = sub.start
        sub.start = self.start
        return sub


def test_hazard_chain_is_correct_and_bit_identical_however_it_is_issued(summary):
    ch = Chain(seed=5)
    plans = [plan_of(case_from_desc(d)) for k, d, _ in ch.launches if k == "igemm"]
    assert plans[0]["ks"] > 1 and plans[1]["ks"] > 1, "launches 1 and 2 must plan split-K"
    assert plans[2]["cluster"] > 1, "launch 3 must exchange pixel-norm statistics through a cluster"
    sub = ch.subject(ch.program())

    # the serialized replay is a correct computation: every launch against fp64 from what it actually read
    sub.reset()
    trace = []
    serialized(sub, trace)
    for i, check in enumerate(ch.checks):
        kind = ch.launches[i][0]

        def note(what, value, i=i, kind=kind):
            _note(summary, what, value, f"launch {i} {kind}")
            assert value <= 1.0, f"launch {i} ({kind}): {what} = {value:.3f}"
        check(trace[i], trace[i + 1], note)
    want = trace[-1]
    unwritten = sub.order([k for k in sub.nan if torch.isnan(want[k].float()).any()])
    assert not unwritten, unwritten
    # ... and every way of issuing it gives the same bits
    modes = compare_modes(sub, want)
    summary["compared"].append((sub.name, len(sub.launches), modes))


def test_hazard_chain_eager_run_issues_each_launch_once():
    """The kernels an eager run puts on the device, in order, are the recorded launches: none dropped, none issued
    twice (a repeated launch of a layer that does not read its own output would not change any buffer)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    ch = Chain(seed=6)
    sub = ch.subject(ch.program())
    sub.reset()
    mode_eager(sub)                   # one run outside the profiler first
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mode_eager(sub)
        torch.cuda.synchronize()
    events = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA),
                    key=lambda e: e.time_range.start)
    issued = []
    for e in events:
        kinds = [kind for key, kind in KERNEL_KIND.items() if key in e.name]
        if kinds:
            issued.append(kinds[0])
    assert issued == [k for k, _, _ in ch.launches], issued


# ------------------------------------------------------------------------------------------------ the program API
def _serialized_state(ch):
    sub = ch.subject(ch.program(upto=0))
    sub.reset()
    serialized(sub)
    return sub, sub.snapshot()


def test_add_copies_the_descriptor_and_the_embed_block_array():
    ch, decoy = Chain(seed=7), Chain(seed=8)
    ref_sub, want = _serialized_state(ch)
    decoy_sub = decoy.subject(decoy.program(upto=0), "decoy")
    decoy_sub.reset()
    decoy_start = decoy_sub.snapshot()
    # add copies of the chain's descriptors (and block arrays), then overwrite every copy with the decoy chain's
    # descriptor, pointing at other, valid buffers: the program must still run the chain as it was added
    prog = UNetProgram(DEV)
    added = []
    for (kind, d, _), (_, dd, _) in zip(ch.launches, decoy.launches):
        mine = type(d).from_buffer_copy(d)
        arr = None
        if kind == "embed":
            arr = (L.TdxEmbedBlock * d.n_blocks)()
            C.memmove(arr, d.blocks, C.sizeof(arr))
            mine.blocks = arr
        L.check(getattr(L.lib(), f"tdx_program_add_{kind}")(prog.handle, C.byref(mine)))
        if arr is not None:
            C.memmove(arr, dd.blocks, C.sizeof(arr))
        C.memmove(C.addressof(mine), C.addressof(dd), C.sizeof(mine))
        added.append((mine, arr))
    sub = ch.subject(prog)
    for mode, run in (("graph", mode_graph), ("eager", mode_eager)):
        sub.reset()
        run(sub)
        torch.cuda.synchronize()
        assert_identical(sub, sub.snapshot(), want, f"{mode}, descriptors overwritten after add")
        assert_identical(decoy_sub, decoy_sub.snapshot(), decoy_start, f"{mode}: the decoy buffers")
    # a program whose descriptors and block arrays are dropped right after each add
    prog2 = UNetProgram(DEV)
    for kind, d, _ in ch.launches:
        mine = type(d).from_buffer_copy(d)
        if kind == "embed":
            arr = (L.TdxEmbedBlock * d.n_blocks)()
            C.memmove(arr, d.blocks, C.sizeof(arr))
            mine.blocks = arr
            del arr
        L.check(getattr(L.lib(), f"tdx_program_add_{kind}")(prog2.handle, C.byref(mine)))
        del mine
    gc.collect()
    sub2 = ch.subject(prog2)
    sub2.reset()
    mode_graph(sub2)
    torch.cuda.synchronize()
    assert_identical(sub2, sub2.snapshot(), want, "graph, descriptors dropped after add")


def test_add_after_the_graph_exists_captures_again():
    ch = Chain(seed=9)
    _, want = _serialized_state(ch)
    n = len(ch.launches)
    prog = ch.program(upto=n - 1)
    sub = ch.subject(prog)
    sub.reset()
    mode_graph(sub)
    torch.cuda.synchronize()
    assert L.lib().tdx_program_num_launches(prog.handle) == n - 1
    assert torch.isnan(sub.state["y"].float()).all()          # the last launch is not in the program yet
    kind, d, _ = ch.launches[-1]
    L.check(L.lib().tdx_program_add_igemm(prog.handle, C.byref(d)))
    assert L.lib().tdx_program_num_launches(prog.handle) == n
    sub.reset()
    mode_graph(sub)
    torch.cuda.synchronize()
    assert not torch.isnan(sub.state["y"].float()).any(), "the launch added after the first capture did not run"
    assert_identical(sub, sub.snapshot(), want, "graph, after a late add")


def test_failed_add_leaves_the_program_unchanged():
    ch = Chain(seed=10)
    _, want = _serialized_state(ch)
    prog = ch.program()
    sub = ch.subject(prog)
    sub.reset()
    mode_graph(sub)
    torch.cuda.synchronize()
    n = len(ch.launches)
    bad_ig = L.TdxIgemmDesc.from_buffer_copy(ch.launches[1][1])
    bad_ig.n_seg = 0
    bad_em = L.TdxEmbedDesc.from_buffer_copy(ch.launches[0][1])
    bad_em.n_blocks = 0
    for fn, d, field in ((L.lib().tdx_program_add_igemm, bad_ig, "n_seg"),
                         (L.lib().tdx_program_add_embed, bad_em, "n_blocks")):
        assert fn(prog.handle, C.byref(d)) == -1                  # TDX_E_INVALID
        assert field in L.lib().tdx_last_error().decode()
        assert L.lib().tdx_program_num_launches(prog.handle) == n
    sub.reset()
    mode_graph(sub)
    torch.cuda.synchronize()
    assert_identical(sub, sub.snapshot(), want, "graph, after failed adds")


def test_graph_fixes_addresses_not_contents():
    ch = Chain(seed=11)
    prog = ch.program()
    sub = ch.subject(prog)
    sub.reset()
    mode_graph(sub)
    torch.cuda.synchronize()
    first = sub.snapshot()
    # new values in the same input buffers
    g = torch.Generator(device=DEV).manual_seed(99)
    for k in ("emb_a", "emb_b", "sample", "x0_prev"):
        sub.start[k] = torch.randn(sub.start[k].shape, generator=g, device=DEV)
    sub.start["x"] = _nc8(Chain.C, g, DEV)
    sub.start["c_in"].fill_(1.7)
    sub.reset()
    serialized(sub)
    want = sub.snapshot()
    assert not _same_bits(want["y"], first["y"])
    sub.reset()
    mode_graph(sub)
    torch.cuda.synchronize()
    assert_identical(sub, sub.snapshot(), want, "graph, new input values")


def test_instantiate_on_one_stream_and_run_on_another():
    ch = Chain(seed=12)
    _, want = _serialized_state(ch)
    prog = ch.program()
    sub = ch.subject(prog)
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    with torch.cuda.stream(s1):
        L.call(L.lib().tdx_program_instantiate, DEV, prog.handle)
    s1.synchronize()
    sub.reset()
    s2.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s2):
        L.call(L.lib().tdx_program_run, DEV, prog.handle, 1)
    s2.synchronize()
    assert_identical(sub, sub.snapshot(), want, "instantiated on one stream, run on another")


def test_empty_program_runs_instantiates_and_profiles():
    h = C.c_void_p()
    L.check(L.lib().tdx_program_create(C.byref(h)))
    try:
        assert L.lib().tdx_program_num_launches(h) == 0
        L.call(L.lib().tdx_program_run, DEV, h, 0)
        L.call(L.lib().tdx_program_run, DEV, h, 1)
        L.call(L.lib().tdx_program_instantiate, DEV, h)
        L.call(L.lib().tdx_program_run, DEV, h, 1)
        ms, kinds = (C.c_float * 1)(-1.0), (C.c_int32 * 1)(-7)
        L.call(L.lib().tdx_program_profile, DEV, h, ms, kinds)
        assert ms[0] == -1.0 and kinds[0] == -7           # nothing to report, nothing written
        torch.cuda.synchronize()
    finally:
        assert L.lib().tdx_program_destroy(h) == 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_program_for_the_second_device_runs_while_the_first_is_current():
    dev1 = torch.device("cuda:1")
    with torch.cuda.device(dev1):
        ch = Chain(seed=13, device=dev1)
        prog = ch.program()
        sub = ch.subject(prog)
        sub.reset()
        serialized(sub)
        want = sub.snapshot()
        sub.reset()
        torch.cuda.synchronize(dev1)
    with torch.cuda.device(0):
        assert torch.cuda.current_device() == 0
        L.call(L.lib().tdx_program_run, dev1, prog.handle, 1)
    torch.cuda.synchronize(dev1)
    assert_identical(sub, sub.snapshot(), want, "graph on cuda:1 while cuda:0 is current")
