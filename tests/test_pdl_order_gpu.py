"""Every libtdx kernel waits for its predecessor before it touches what that predecessor reads or writes.

Under programmatic dependent launch (PDL) a kernel may start while the kernel before it on the stream is still running;
only pdl_wait() (griddepcontrol.wait) orders it after that kernel.  Torch kernels never trigger an early launch, so a
test that writes its inputs with torch and then calls an entry point never runs a libtdx kernel beside a predecessor
that is still writing.  Here the predecessor is the debug hook tdx_debug_pdl_interpose (csrc/tdx_debug_pdl.cu): a
small kernel that poisons a set of regions, lets the next launch start, spins for DELAY_NS, snapshots the regions and
restores them.  A successor that waits sees the original data; one that reads a region early computes from the poison,
and one that writes a region early leaves its write in the snapshot.

Every entry point.  Each case of tests/test_input_extents_gpu.py (every entry point, at edge and product shapes) runs
plainly, then twice with L.lib() wrapped in a proxy that issues the interposer on the call's stream before every
kernel-launching tdx_* call.  The interposer covers every device input and every output the case has registered so
far, with the poison of the buffer's role (tests/_fence.py):

    role               pattern A            pattern B
    fp32, fp64, bf16   NaN                  1e30
    int                0x00 bytes           0xFF bytes
    index              index_values[0]      index_values[1]

except TdxIgemmDesc.b_packed and TdxConvOutDesc.weight, which tdx.h allows those kernels to read before they wait,
and scratch outputs, which are snapshotted but not poisoned.  Asserted: every compared output is byte-identical to the
plain run, every snapshot holds exactly the poison (the original contents for scratch), inputs and guards are intact.

These entry points run a memset before their first kernel, so the stream, not PDL, orders that kernel after the
interposer and nothing overlaps it: tdx_flow_d8, tdx_flow_link, tdx_flow_accumulate, tdx_relief_stats,
tdx_detail_range, tdx_coarse_readout, tdx_noise_patch, tdx_noise_patches and tdx_standard_normal (and tdx_coarse_land
when no window fits, where the memset is all it does).  Their later kernels, and the second and later kernels of every
multi-kernel entry point, are covered by the static rule of tests/test_launch_policy_cpu.py, not here.

Every shipped program, launch by launch.  Each program of tests/test_program_gpu.py is replayed with every recorded
descriptor through its own entry point and an interposer in place of the synchronise between launches, poisoning and
snapshotting the whole program state except that launch's b_packed or conv_out weight.  So launch i+1 runs against a
launch i that finishes late, for every launch of the decoder, base, coarse, solve and autoencoder programs.  The
final state must equal the serialized replay bit for bit and every snapshot must hold the poison.

Controls.  Without them a run in which nothing overlapped would pass silently: one product igemm launch with b_packed
poisoned and one multi-CTA conv_out launch with weight poisoned must change their outputs (both read these before
they wait).  Each runs once.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import struct
import time

import numpy as np
import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from tests import _igemm_ref as IR
from tests import test_input_extents_gpu as IE
from tests import test_program_gpu as TP
from tests._igemm_surface import product_representatives
from tests.test_entry_points_cpu import header_entry_points

pytestmark = pytest.mark.gpu

DEV = IE.DEV
DELAY_NS = 1_000_000
"""How long the interposer holds its regions poisoned after it lets the successor start.  The successor has to be
enqueued by the host and become resident inside this window; the controls show that it does."""
POISONS = ("A", "B")
EARLY = {"TdxIgemmDesc.b_packed", "TdxConvOutDesc.weight"}
"""Inputs tdx.h allows a kernel to read before it waits (the igemm weights, the conv_out weights)."""

NOT_LAUNCHING = {
    "tdx_last_error", "tdx_device_info", "tdx_abi_sizeof",                             # queries
    "tdx_igemm_choose_n", "tdx_igemm_packed_weight_elems",
    "tdx_noise_patch_workspace_bytes", "tdx_noise_patches_workspace_bytes",            # workspace sizes
    "tdx_tile_seed",                                                                   # host-side hash
    "tdx_noise_patch_status",                                                          # synchronises and reads a flag
    "tdx_program_create", "tdx_program_add_im2col", "tdx_program_add_igemm", "tdx_program_add_conv_out",
    "tdx_program_add_embed", "tdx_program_add_attn", "tdx_program_num_launches", "tdx_program_destroy",
    "tdx_program_instantiate",                                                         # captures and uploads, runs none
}
LAUNCHING = header_entry_points() - NOT_LAUNCHING

_F32_BIG = struct.unpack("<I", struct.pack("<f", 1e30))[0]
_F64_BIG = struct.unpack("<Q", struct.pack("<d", 1e30))[0]
POISON_WORD = {     # role -> pattern -> (bytes, word); the index role takes its word from the buffer's index_values
    "f32": {"A": (4, 0x7FC00000), "B": (4, _F32_BIG)},
    "f64": {"A": (8, 0x7FF8000000000000), "B": (8, _F64_BIG)},
    "bf16": {"A": (2, 0x7FC0), "B": (2, _F32_BIG >> 16)},
    "int": {"A": (1, 0x00), "B": (1, 0xFF)},
}


def poison_word(role, dtype, pattern, index_values=(-1, 0)):
    if role == "index":
        esz = torch.empty((), dtype=dtype).element_size()
        v = index_values[0 if pattern == "A" else 1]
        return esz, v & ((1 << (8 * esz)) - 1)
    return POISON_WORD[role][pattern]


def _signed(v):
    return v - (1 << 64) if v >= 1 << 63 else v


def _interpose_fn():
    fn = L.lib().tdx_debug_pdl_interpose
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_void_p]
    return fn


class Region:
    """ptr, bytes and the poison word (bytes, value) of one device buffer; word bytes 0: scratch, not poisoned."""

    def __init__(self, name, ptr, nbytes, word=(0, 0)):
        self.name, self.ptr, self.nbytes, self.word = name, ptr, nbytes, word
        assert word[0] == 0 or nbytes % word[0] == 0, (name, nbytes, word)

    def expected(self, save):
        """The bytes the snapshot must hold: the poison, or the saved contents of a scratch buffer."""
        if self.word[0] == 0:
            return save
        pat = torch.tensor(list(self.word[1].to_bytes(self.word[0], "little")), dtype=torch.uint8, device=DEV)
        return pat.repeat(self.nbytes // self.word[0])


class Issued:
    """One interposer launch: its region table, save and snapshot buffers (kept alive until checked)."""

    def __init__(self, regions, stream):
        self.regions = regions
        self.save = [torch.empty(max(r.nbytes, 16), dtype=torch.uint8, device=DEV) for r in regions]
        self.snap = [torch.empty(max(r.nbytes, 16), dtype=torch.uint8, device=DEV) for r in regions]
        rows = [[r.ptr, r.nbytes, _signed(r.word[1]), r.word[0], s.data_ptr(), p.data_ptr()]
                for r, s, p in zip(regions, self.save, self.snap)]
        self.table = torch.tensor(rows or [[0] * 6], dtype=torch.int64).pin_memory().to(DEV, non_blocking=True)
        L.check(_interpose_fn()(self.table.data_ptr(), len(regions), DELAY_NS, stream))

    def bad(self):
        """[(region name, bytes that differ from what the snapshot must hold)] after a synchronise."""
        out = []
        for r, s, p in zip(self.regions, self.save, self.snap):
            n = int((p[:r.nbytes] != r.expected(s[:r.nbytes])).sum())
            if n:
                out.append((r.name, n))
        return out


class Proxy:
    """Stands in for the loaded library: before every kernel-launching tdx_* call, `before(name, stream)` runs."""

    def __init__(self, lib, before):
        self.lib, self.before = lib, before

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if name not in LAUNCHING:
            return fn

        def interposed(*args):
            self.before(name, args[-1])
            return fn(*args)
        return interposed


@contextlib.contextmanager
def interposing(before):
    real = L.lib
    proxy = Proxy(real(), before)
    L.lib = lambda: proxy
    try:
        yield
    finally:
        L.lib = real


REACHED: set = set()       # launching entry points reached through an interposed call
STATS = {"cases": {}, "programs": [], "controls": [], "t0": None}


@pytest.fixture(scope="module", autouse=True)
def summary(request):
    STATS["t0"] = time.perf_counter()
    yield
    wall = time.perf_counter() - STATS["t0"]
    lines = [f"interposed {e}: {n} cases" for e, n in sorted(STATS["cases"].items())]
    lines += [f"program {name}: {n} launches replayed interposed, bit-identical under patterns {', '.join(POISONS)}"
              for name, n in STATS["programs"]]
    lines += [f"control {what}: {n} of {total} output elements changed" for what, n, total in STATS["controls"]]
    n_cases = sum(STATS["cases"].values())
    n_launch = sum(n for _, n in STATS["programs"])
    lines.append(f"pdl order: {n_cases} cases and {n_launch} program launches interposed (delay {DELAY_NS / 1e3:.0f} us"
                 f" each, per pattern) in {wall:.1f} s wall")
    IR.report(request.config, lines)


# ------------------------------------------------------------------------------------------------ entry points
class PoisonEnv(IE.Env):
    """An Env that also remembers each input's index_values, so that index data is poisoned with valid indices."""

    def __init__(self, entry, pattern, poison_early=False):
        super().__init__(entry, pattern)
        self.index_values, self.poison_early, self.issued = {}, poison_early, []

    def inp(self, name, data, role=None, host=False, pitch=None, index_values=(-1, 0)):
        f = super().inp(name, data, role, host, pitch, index_values)
        self.index_values[id(f)] = index_values
        return f

    def regions(self):
        out = []
        for name, f in self.inputs:
            if not isinstance(f, IE.Fenced) or f.host or (name in EARLY and not self.poison_early):
                continue
            word = poison_word(f.role, f.dtype, self.pattern, self.index_values[id(f)])
            out.append(Region(name, f.raw.data_ptr() + f.fence, f.body_bytes, word))
        for name, (g, compare) in self.outputs.items():
            v = g.view
            role = IE._DEFAULT_ROLE.get(v.dtype, "int")
            word = poison_word(role, v.dtype, self.pattern) if compare else (0, 0)
            out.append(Region(name, v.data_ptr(), v.numel() * v.element_size(), word))
        return out

    def before(self, name, stream):
        REACHED.add(name)
        self.issued.append((name, Issued(self.regions(), stream)))


def _run(case, pattern, poison_early=False):
    env = PoisonEnv(case.entry, pattern, poison_early)
    if pattern is None:
        case.fn(env)
    else:
        with interposing(env.before):
            case.fn(env)
    torch.cuda.synchronize()
    tag = f"{case.name} [{'plain' if pattern is None else 'poison ' + pattern}]"
    for name, f in env.inputs:
        if f is not None:
            assert f.unchanged(), f"{tag}: input {name} (or its fence) changed"
    for name, (g, _) in env.outputs.items():
        g.check(f"{tag}: {name}")
    for i, (fn, iss) in enumerate(env.issued):
        bad = iss.bad()
        assert not bad, f"{tag}: call {i} ({fn}) wrote before it waited: {bad}"
    return env, {k: IE._as_bytes(v) for k, v in env.snapshot().items()}


def run_interposed(case):
    _, base = _run(case, None)
    assert base, f"{case.name}: nothing compared"
    changed, issued = [], 0
    for pattern in POISONS:
        env, got = _run(case, pattern)
        issued += len(env.issued)
        assert got.keys() == base.keys()
        diff = [k for k in base if got[k] != base[k]]
        if diff:
            changed.append(f"poison {pattern} changed {diff}")
    assert not changed, f"{case.name}: {'; '.join(changed)}: a kernel read its inputs before it waited"
    if issued:
        STATS["cases"][case.entry] = STATS["cases"].get(case.entry, 0) + 1


EXTRA: list = []


def extra(entry):
    def deco(fn):
        EXTRA.append(IE.Case(f"{entry}[small]", entry, fn))
        return fn
    return deco


@extra("tdx_noise_patch")
def _noise_patch(env):
    nb = L.lib().tdx_noise_patch_workspace_bytes(2, 64, 64)
    ws = env.out("workspace", (nb,), torch.uint8, compare=False)
    ws.view.zero_()
    o = env.out("out", (2, 33, 37))
    IE.call("tdx_noise_patch", 777, -37, 91, 33, 37, 2, 64, 64, o.data_ptr(), ws.data_ptr(), nb)


@extra("tdx_standard_normal")
def _standard_normal(env):
    n = 1000
    nb = L.lib().tdx_noise_patch_workspace_bytes(1, 1, n)
    ws = env.out("workspace", (nb,), torch.uint8, compare=False)
    ws.view.zero_()
    o = env.out("out", (n,))
    IE.call("tdx_standard_normal", 4321, n, o.data_ptr(), ws.data_ptr(), nb)


def pytest_generate_tests(metafunc):
    if metafunc.function.__name__ == "test_entry_point_waits_for_its_predecessor":
        IE._gpu_run[0] = IE.gpu_tests_selected(metafunc.config)
        cases = IE.CASES + IE.igemm_cases() + EXTRA
        metafunc.parametrize("c", cases, ids=[c.name for c in cases])


def test_entry_point_waits_for_its_predecessor(c):
    run_interposed(c)


# ------------------------------------------------------------------------------------------------ programs
class StateRegions:
    """The program state as disjoint regions in flat save / snapshot buffers; each launch's table leaves out its own
    b_packed / conv_out weight."""

    def __init__(self, sub, pattern):
        spans = sorted((t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), t.element_size(), k, t)
                       for k, t in sub.state.items())
        merged = []
        for lo, hi, esz, k, t in spans:
            assert t.is_contiguous(), k
            if merged and lo < merged[-1][1]:
                m = merged[-1]
                merged[-1] = [m[0], max(m[1], hi), min(m[2], esz), m[3], m[4] if m[2] <= esz else t]
            else:
                merged.append([lo, hi, esz, k, t])
        self.regions, offs, total = [], [], 0
        for lo, hi, _, k, t in merged:
            role = IE._DEFAULT_ROLE.get(t.dtype, "int")
            self.regions.append(Region(k, lo, hi - lo, poison_word(role, t.dtype, pattern)))
            offs.append(total)
            total += -(-(hi - lo) // 16) * 16
        self.save = torch.empty(max(total, 16), dtype=torch.uint8, device=DEV)
        self.expect = torch.empty_like(self.save)
        for r, o in zip(self.regions, offs):
            self.expect[o:o + r.nbytes] = r.expected(None)
        self.snap = self.expect.clone()
        self.offs = offs
        rows = []
        for kind, d, _ in sub.launches:
            early = d.b_packed if kind == "igemm" else (d.weight if kind == "conv_out" else None)
            rows.append([[r.ptr, r.nbytes, _signed(r.word[1]), r.word[0], self.save.data_ptr() + o,
                          self.snap.data_ptr() + o]
                         for r, o in zip(self.regions, offs) if not (early and r.ptr <= early < r.ptr + r.nbytes)])
        width = max(len(x) for x in rows)
        self.counts = [len(x) for x in rows]
        self.table = torch.tensor([x + [[0] * 6] * (width - len(x)) for x in rows], dtype=torch.int64).to(DEV)

    def first_bad(self):
        bad = [r.name for r, o in zip(self.regions, self.offs)
               if not torch.equal(self.snap[o:o + r.nbytes], self.expect[o:o + r.nbytes])]
        return bad


def replay_interposed(sub, pattern):
    """Every recorded descriptor through its own entry point, an interposer before each instead of a synchronise;
    returns the launches after which a snapshot did not hold the poison."""
    st = StateRegions(sub, pattern)
    bad = torch.zeros(len(sub.launches), dtype=torch.int64, device=DEV)
    interpose = _interpose_fn()
    sub.reset()
    torch.cuda.synchronize()
    stream = L.current_stream_ptr(sub.device)
    for i, (kind, d, _) in enumerate(sub.launches):
        row = st.table[i]
        L.check(interpose(row.data_ptr(), st.counts[i], DELAY_NS, stream))
        L.check(getattr(L.lib(), f"tdx_{kind}_run")(C.byref(d), stream))
        bad[i] = (st.snap != st.expect).sum()
        st.snap.copy_(st.expect)
    torch.cuda.synchronize()
    return [i for i in range(len(sub.launches)) if int(bad[i])]


@pytest.mark.parametrize("name", TP.PROGRAMS)
def test_program_launches_wait_for_their_predecessor(name, monkeypatch):
    sub = TP.build_subject(name, monkeypatch)
    want = TP.serialized_reference(sub)
    for pattern in POISONS:
        early = replay_interposed(sub, pattern)
        assert not early, (f"{name}, poison {pattern}: launches that wrote program state before they waited: "
                           f"{[(i, sub.launches[i][0]) for i in early[:12]]}")
        TP.assert_identical(sub, sub.snapshot(), want, f"interposed, poison {pattern}")
    STATS["programs"].append((name, len(sub.launches)))


@pytest.mark.parametrize("entry", ["tdx_program_run", "tdx_program_profile"])
def test_program_entry_points_wait_for_their_predecessor(entry):
    """tdx_program_run(use_graph=0) and tdx_program_profile on the hand-built hazard chain, the interposer in front
    of the call covering the chain's whole state."""
    ch = TP.Chain(seed=5)
    sub = ch.subject(ch.program())

    def run():
        if entry == "tdx_program_run":
            TP.mode_eager(sub)
        else:
            TP.mode_profile(sub)
        torch.cuda.synchronize()
    sub.reset()
    torch.cuda.synchronize()
    run()
    want = sub.snapshot()
    for pattern in POISONS:
        regions = StateRegions(sub, pattern).regions
        issued = []

        def before(fn, stream):
            REACHED.add(fn)
            issued.append(Issued(regions, stream))
        sub.reset()
        torch.cuda.synchronize()
        with interposing(before):
            run()
        assert len(issued) == 1
        bad = issued[0].bad()
        assert not bad, f"{entry}, poison {pattern}: the first launch wrote before it waited: {bad}"
        TP.assert_identical(sub, sub.snapshot(), want, f"{entry} interposed, poison {pattern}")
    STATS["cases"][entry] = STATS["cases"].get(entry, 0) + 1


# ------------------------------------------------------------------------------------------------ controls
def _changed(a: bytes, b: bytes, esz: int) -> int:
    x = np.frombuffer(a, dtype=np.uint8).reshape(-1, esz)
    y = np.frombuffer(b, dtype=np.uint8).reshape(-1, esz)
    return int((x != y).any(axis=1).sum())


def _control(case, key, esz, what):
    _, base = _run(case, None)
    _, got = _run(case, "A", poison_early=True)
    n, total = _changed(got[key], base[key], esz), len(base[key]) // esz
    STATS["controls"].append((what, n, total))
    assert n > 0, f"{what}: the interposer did not overlap its successor; nothing here was tested"


def test_control_igemm_reads_its_weights_before_it_waits():
    c = product_representatives()[0]
    case = IE.Case(f"tdx_igemm_run[{c.name}]", "tdx_igemm_run", lambda env: IE.igemm_case(c, env))
    _control(case, "out0", 2, f"igemm {c.name} with b_packed poisoned")


def test_control_conv_out_reads_its_weights_before_it_waits():
    case = next(x for x in IE.CASES if x.name == "tdx_conv_out_run[1,64,64,192,5,1]")
    _control(case, "model_out", 4, "conv_out 1x192x64x64 -> 5 with weight poisoned")


# ------------------------------------------------------------------------------------------------ coverage
def test_every_launching_entry_point_was_interposed(request):
    """Runs last: every kernel-launching entry point of tdx.h was reached through an interposed call."""
    assert "tdx_igemm_run" in LAUNCHING and "tdx_program_run" in LAUNCHING
    assert not NOT_LAUNCHING - header_entry_points(), sorted(NOT_LAUNCHING - header_entry_points())
    ran = {i.originalname for i in request.session.items if i.module is request.module}
    n_cases = sum(1 for i in request.session.items if i.originalname == "test_entry_point_waits_for_its_predecessor")
    if n_cases < len(IE.CASES + IE.igemm_cases() + EXTRA) or not {"test_program_entry_points_wait_for_their_predecessor",
                                                                 "test_program_launches_wait_for_their_predecessor"} <= ran:
        pytest.skip("only some cases ran")
    missing = sorted(LAUNCHING - REACHED)
    assert not missing, f"kernel-launching entry points no interposed call reached: {missing}"
