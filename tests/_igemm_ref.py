"""Plain-PyTorch fp64 reference of ONE tdx_igemm_run launch (conv + fused epilogue), and a runner for the CUDA op.

Used by tests/test_igemm_gpu.py, tests/test_igemm_plans_gpu.py and tools/bringup_igemm.py.  Inputs are rounded to bf16
first so that the only difference to the kernel is accumulation order and the bf16 rounding of the stored outputs.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.layout import from_nc8hw8, pack_weight_segments, to_nc8hw8

TILE_H, TILE_W = 16, 8          # pixels of one work item (kTileH x kTileW in tdx_igemm.cu)
GUARD_BYTES = 4096              # sentinel before and after every output buffer
SENTINEL16, SENTINEL32 = 0x5A5B, 0x5A5B5C5D


def mp_silu(x):
    return F.silu(x) / 0.596


def pixelnorm(x):
    return x / (1e-4 + x.square().mean(dim=1, keepdim=True).sqrt())


@dataclass
class Case:
    name: str
    segs: list  # [(channels, taps)]
    cout: int
    n: int
    h: int
    w: int
    epi: int = 0
    resid_spatial: int = L.SP_SAME
    resid_pnorm: int = 0
    resid_scale: float = 0.7
    clip: float = 0.0
    outs: list = field(default_factory=lambda: [(L.OUT_RAW, L.SP_SAME, 1.0)])
    wscale: float = 1.0
    n_item: int = 0   # 0 = let the library choose (tdx_igemm_choose_n)
    seed: int = 0
    rms_out: bool = False     # the launch also stores 1 / (eps + rms) of its result per pixel
    resid_inv: bool = False   # the residual's pixel-norm comes from a precomputed plane (needs resid_pnorm)

    @property
    def macs(self) -> int:
        return self.n * self.h * self.w * self.cout * sum(c * t for c, t in self.segs)


def case_from_desc(d, name: str = "desc", seed: int = 0) -> Case:
    """The Case that replays descriptor `d` (a TdxIgemmDesc recorded from the product) with fresh inputs: same segments,
    shape, work-item width, epilogue, residual mode, pixel-norm side planes, scale, clip and outputs."""
    segs = [(int(d.a_channels[i]), int(d.a_taps[i])) for i in range(d.n_seg)]
    outs = [(int(o.kind), int(o.spatial), float(o.scale)) for o in d.out if o.kind != L.OUT_NONE]
    resid_inv = bool(d.resid_inv)
    return Case(name, segs, int(d.c_out), int(d.n_img), int(d.height), int(d.width), epi=int(d.epi_flags),
                resid_spatial=int(d.resid_spatial), resid_pnorm=1 if resid_inv else int(d.resid_pnorm),
                resid_scale=float(d.resid_scale), clip=float(d.clip), outs=outs, n_item=int(d.n_per_item), seed=seed,
                rms_out=bool(d.rms_out), resid_inv=resid_inv)


def needs_norm(case: Case) -> bool:
    """Whether the launch computes per-pixel statistics over all c_out channels (as igemm_launch decides it)."""
    return bool(case.epi & L.EPI_PNORM) or case.rms_out or any(k == L.OUT_PNORM_SILU for k, _, _ in case.outs)


def device_sm_count() -> int:
    sm, ma, mi = C.c_int(), C.c_int(), C.c_int()
    L.check(L.lib().tdx_device_info(C.byref(sm), C.byref(ma), C.byref(mi)))
    return sm.value


def plan_of(case: Case, sm_count: int | None = None) -> dict:
    """The launch plan igemm_launch makes for this case on the current device: work-item width N, split-K factor,
    resident weights or ring depth SB, cluster size, and the grid it derives from them (rounds = work items per CTA,
    `partial` = the last round leaves some CTAs idle).  `ragged` = the height is not a multiple of the 16-row tile.
    `ov` = igemm_launch runs it on the overlapped-epilogue kernel (its `overlapped()`: cluster-free, N <= 128, more
    than one round, no pixel-norm statistics), otherwise on the serial-epilogue kernel."""
    ch = (C.c_int32 * 3)(*[c for c, _ in case.segs], *([0] * (3 - len(case.segs))))
    tp = (C.c_int32 * 3)(*[t for _, t in case.segs], *([0] * (3 - len(case.segs))))
    n_item = case.n_item or L.igemm_choose_n(case.cout, case.n, case.h, case.w, case.segs)
    norm = needs_norm(case)
    out = (C.c_int32 * 4)()
    L.lib().tdx_debug_igemm_plan(case.cout, case.n, case.h, case.w, ch, tp, len(case.segs), n_item, int(norm), out)
    N, ks, resident, sb = (int(v) for v in out)
    nsplit = case.cout // N
    cluster = nsplit * ks if (norm and nsplit * ks > 1) else ks
    tiles = -(-case.h // TILE_H) * -(-case.w // TILE_W) * case.n
    items = tiles * nsplit * ks
    sms = device_sm_count() if sm_count is None else sm_count
    grid = min(items, sms)
    grid -= grid % (nsplit * ks)
    rounds = -(-items // grid)
    return dict(N=N, ks=ks, resident=resident, SB=sb, cluster=cluster, nsplit=nsplit, items=items, grid=grid,
                rounds=rounds, partial=items % grid != 0, ragged=case.h % TILE_H != 0,
                ov=cluster == 1 and N <= 128 and rounds > 1 and not norm)


def plan_class(p: dict) -> tuple:
    """(N, ksplit, resident, SB, cluster size, more than one round, ragged): what makes two launches take different
    paths through the kernel."""
    return (p["N"], p["ks"], p["resident"], p["SB"], p["cluster"], p["rounds"] > 1, p["ragged"])


def plan_label(cls: tuple) -> str:
    N, ks, res, sb, cl, multi, ragged = cls
    return (f"N{N}-ks{ks}-{'res' if res else 'SB'}{sb}-cl{cl}-{'multi' if multi else 'one'}"
            f"{'-ragged' if ragged else ''}")


def plan_variant(p: dict) -> tuple:
    """plan_class + (partial last round, overlapped-epilogue kernel): on the overlapped kernel the last round, partial
    or not, is where the MMA warpgroups and the epilogue warpgroup fall out of step."""
    return plan_class(p) + (p["partial"], p["ov"])


def variant_label(v: tuple) -> str:
    *cls, partial, ov = v
    return f"{plan_label(tuple(cls))}{'-partial' if partial else ''}-{'ov' if ov else 'serial'}"


def make_inputs(case: Case, device):
    """bf16-exact activations, weights and residual, fp32 modulation vector (drawn on `device`: a 40-image case takes
    milliseconds)."""
    device = torch.device(device)
    g = torch.Generator(device=device).manual_seed(case.seed)
    acts, wts = [], []
    ktot = sum(c * t for c, t in case.segs)
    for (c, t) in case.segs:
        a = torch.randn(case.n, c, case.h, case.w, generator=g, device=device)
        k = 3 if t == 9 else 1
        w = torch.randn(case.cout, c, k, k, generator=g, device=device) * (case.wscale / ktot ** 0.5)
        acts.append(a.bfloat16().float())
        wts.append(w.bfloat16().float())
    cvec = 1.0 + 0.3 * torch.randn(case.n, case.cout, generator=g, device=device)
    resid = torch.randn(case.n, case.cout, *resid_size(case), generator=g, device=device).bfloat16().float()
    return acts, wts, cvec, resid


def resid_size(case: Case) -> tuple:
    if case.resid_spatial == L.SP_UP2:
        return (case.h // 2, case.w // 2)
    if case.resid_spatial == L.SP_DOWN2:
        return (case.h * 2, case.w * 2)
    return (case.h, case.w)


def reference(case: Case, acts, wts, cvec, resid):
    """fp64 outputs of the launch; with case.rms_out one more entry: the fp64 plane 1 / (eps + rms) of the result."""
    acc = None
    for a, w in zip(acts, wts):
        y = F.conv2d(a.double(), w.double(), padding=w.shape[-1] // 2)
        acc = y if acc is None else acc + y
    v = acc
    if case.epi & L.EPI_EMB_SILU:
        v = mp_silu(v * cvec.double()[:, :, None, None])
    if case.epi & L.EPI_RESID:
        r = resid.double()
        if case.resid_pnorm:
            r = pixelnorm(r)
        if case.resid_spatial == L.SP_UP2:
            r = r.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        elif case.resid_spatial == L.SP_DOWN2:
            r = r[:, :, ::2, ::2]
        v = v + case.resid_scale * r
    if case.clip > 0:
        v = torch.clamp(v, -case.clip, case.clip)
    inv = 1.0 / (1e-4 + v.square().mean(dim=1).sqrt())
    if case.epi & L.EPI_PNORM:
        v = pixelnorm(v)
    outs = []
    for kind, spatial, scale in case.outs:
        if kind == L.OUT_RAW:
            o = v
        elif kind == L.OUT_SILU:
            o = mp_silu(scale * v)
        else:
            o = mp_silu(v if (case.epi & L.EPI_PNORM) else pixelnorm(v))
        if spatial == L.SP_DOWN2:
            o = o[:, :, ::2, ::2]
        elif spatial == L.SP_UP2:
            o = o.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        outs.append(o)
    if case.rms_out:
        outs.append(inv)
    return outs


class Guarded:
    """A tensor view inside a larger allocation with GUARD_BYTES of sentinel on each side: check() fails if the kernel
    wrote outside the view.  The view starts 16-byte aligned and is NaN-filled, so an unwritten element fails too."""

    def __init__(self, shape, dtype, device):
        self.dtype = dtype
        raw = torch.int16 if dtype == torch.bfloat16 else torch.int32
        self.sentinel = SENTINEL16 if dtype == torch.bfloat16 else SENTINEL32
        esz = torch.empty((), dtype=dtype).element_size()
        self.pad = GUARD_BYTES // esz
        numel = 1
        for s in shape:
            numel *= s
        self.numel = numel
        self.raw = torch.full((self.pad + numel + self.pad,), self.sentinel, dtype=raw, device=device)
        self.view = self.raw[self.pad:self.pad + numel].view(dtype).view(*shape)
        self.view.fill_(float("nan"))
        assert self.view.data_ptr() % 16 == 0

    def data_ptr(self):
        return self.view.data_ptr()

    def check(self, what):
        before, after = self.raw[:self.pad], self.raw[self.pad + self.numel:]
        bad = int((before != self.sentinel).sum()) + int((after != self.sentinel).sum())
        assert bad == 0, f"{what}: {bad} elements written outside the tensor"


def run_cuda(case: Case, acts, wts, cvec, resid, rms_out=None, resid_inv=None, place=None):
    """One tdx_igemm_run launch.  Every bf16 output (and, with case.rms_out, the fp32 rms plane, returned last) lives
    in a guarded buffer whose sentinels are checked after the launch.  case.resid_inv: the residual's pixel-norm plane
    is computed here from `resid` and passed as resid_inv.  The rms_out / resid_inv arguments pass caller-owned planes
    instead.  place(name, value), when given, decides where each input lives: it receives every device input in the
    layout the kernel reads ("TdxIgemmDesc.<field>": a tensor) and the filled descriptor ("desc") and returns the tensor
    (or descriptor pointer) to pass instead (tests/test_input_extents_gpu.py fences them)."""
    dev = acts[0].device
    keep = place if place is not None else (lambda name, value: value)
    a_dev = [keep("TdxIgemmDesc.a_ptr", to_nc8hw8(a)) for a in acts]
    n_item = case.n_item or L.igemm_choose_n(case.cout, case.n, case.h, case.w, case.segs)
    b = keep("TdxIgemmDesc.b_packed", pack_weight_segments(wts, n_item).to(dev))
    r_dev = keep("TdxIgemmDesc.resid", to_nc8hw8(resid))
    d = L.TdxIgemmDesc()
    for i, (c, t) in enumerate(case.segs):
        d.a_ptr[i] = a_dev[i].data_ptr()
        d.a_channels[i] = c
        d.a_taps[i] = t
    d.n_seg = len(case.segs)
    d.b_packed = b.data_ptr()
    d.c_out = case.cout
    d.n_per_item = n_item
    d.n_img, d.height, d.width = case.n, case.h, case.w
    d.epi_flags = case.epi
    cvec_dev = keep("TdxIgemmDesc.cvec", cvec.contiguous())
    d.cvec = cvec_dev.data_ptr()
    d.resid = r_dev.data_ptr()
    d.resid_spatial = case.resid_spatial
    if resid_inv is None and case.resid_inv:
        resid_inv = (1.0 / (1e-4 + resid.double().square().mean(dim=1).sqrt())).float().contiguous()
    d.resid_pnorm = case.resid_pnorm if resid_inv is None else 0
    rms_guard = None
    if rms_out is None and case.rms_out:
        rms_guard = Guarded((case.n, case.h, case.w), torch.float32, dev)
        rms_out = rms_guard.view
    if rms_out is not None:        # fp32 [n, h, w]: 1 / (eps + rms) of the result, for the consumer's residual
        d.rms_out = rms_out.data_ptr()
    if resid_inv is not None:      # fp32 plane at the residual's resolution: replaces the recomputed pixel-norm
        resid_inv = keep("TdxIgemmDesc.resid_inv", resid_inv)
        d.resid_inv = resid_inv.data_ptr()
    d.resid_scale = case.resid_scale
    d.clip = case.clip
    bufs = []
    for i, (kind, spatial, scale) in enumerate(case.outs):
        hh, ww = case.h, case.w
        if spatial == L.SP_DOWN2:
            hh, ww = hh // 2, ww // 2
        elif spatial == L.SP_UP2:
            hh, ww = hh * 2, ww * 2
        o = Guarded((case.n, case.cout // 8, hh, ww, 8), torch.bfloat16, dev)
        bufs.append(o)
        d.out[i].ptr = o.data_ptr()
        d.out[i].kind = kind
        d.out[i].spatial = spatial
        d.out[i].scale = scale
    L.call(L.lib().tdx_igemm_run, dev, C.byref(d) if place is None else place("desc", d))
    torch.cuda.synchronize()
    for i, o in enumerate(bufs):
        o.check(f"{case.name} out{i}")
    res = [from_nc8hw8(o.view) for o in bufs]
    if rms_guard is not None:
        rms_guard.check(f"{case.name} rms_out")
        res.append(rms_guard.view.clone())
    return res


def report(config, lines):
    """Write `lines` to the terminal past pytest's output capture, so summaries show under `pytest -q` too."""
    tr = config.pluginmanager.get_plugin("terminalreporter")
    capman = config.pluginmanager.get_plugin("capturemanager")
    if tr is None or capman is None:
        print("\n".join(lines))
        return
    with capman.global_and_fixture_disabled():
        tr.write("\n")                      # off the line of progress dots
        for line in lines:
            tr.write_line(line)


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def elementwise_ratio(got, ref) -> float:
    """max over elements of |got - ref| / (2^-7 |ref| + 2^-12 rms(ref)), ref in fp64: one bf16 ulp (twice the worst
    rounding error, room for a rounding flip after fp32 accumulation) plus a floor for cancellation in the residual
    sum.  <= 1 passes; NaN anywhere in `got` fails."""
    ref = ref.double()
    err = (got.double() - ref).abs()
    bound = 2.0 ** -7 * ref.abs() + 2.0 ** -12 * float(ref.square().mean().sqrt())
    if torch.isnan(err).any():
        return float("inf")
    return float((err / bound).max())


def check_case(case: Case, device, margins: dict | None = None):
    """Run `case` on the GPU against the fp64 reference: rel-RMS < 2e-3 against the bf16-rounded reference and the
    per-element bound of elementwise_ratio on every output (and the rms plane).  Returns the worst ratio."""
    acts, wts, cvec, resid = make_inputs(case, device)
    refs = reference(case, acts, wts, cvec, resid)
    gots = run_cuda(case, acts, wts, cvec, resid)
    worst = 0.0
    for i, (g, r) in enumerate(zip(gots, refs)):
        what = f"{case.name} {'rms_out' if i == len(case.outs) else f'out{i}'}"
        assert not torch.isnan(g).any(), f"{what}: unwritten (NaN) elements"
        if i < len(case.outs):
            assert rel_rms(g, r.bfloat16().double()) < 2e-3, what
        ratio = elementwise_ratio(g, r)
        worst = max(worst, ratio)
        assert ratio <= 1.0, f"{what}: error {ratio:.2f}x the per-element bound"
    if margins is not None:
        margins[case.name] = worst
    return worst


def default_cases() -> list[Case]:
    E, R, P = L.EPI_EMB_SILU, L.EPI_RESID, L.EPI_PNORM
    return [
        Case("c64_3x3_32x32", [(64, 9)], 64, 1, 32, 32),
        Case("c64_3x3_16x8_single_tile", [(64, 9)], 64, 1, 16, 8),
        Case("c64_3x3_8x8_partial_tile", [(64, 9)], 64, 2, 8, 8),
        Case("c64_1x1_32x32", [(64, 1)], 128, 1, 32, 32),
        Case("c128_3x3_64x64_n2", [(128, 9)], 128, 2, 64, 64),
        Case("c192_3x3_32x32", [(192, 9)], 192, 1, 32, 32),
        Case("c256_3x3_32x32", [(256, 9)], 256, 1, 32, 32),
        Case("c64_3x3_256x256", [(64, 9)], 64, 1, 256, 256),
        Case("concat_256+192_to_192_64x64", [(256, 9), (192, 9)], 192, 1, 64, 64),
        Case("res1+skip_3seg", [(64, 9), (128, 1), (64, 1)], 64, 1, 64, 64),
        Case("emb_silu", [(64, 9)], 64, 2, 32, 32, epi=E),
        Case("resid_same_pnorm_3outs", [(128, 9)], 128, 1, 32, 32, epi=R, resid_pnorm=1,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_SAME, 1.0), (L.OUT_SILU, L.SP_SAME, 0.83)]),
        Case("resid_down_pnorm_down2", [(64, 9)], 64, 1, 32, 32, epi=R, resid_spatial=L.SP_DOWN2, resid_pnorm=1,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_DOWN2, 1.0)]),
        Case("resid_up_up2", [(128, 9)], 128, 1, 32, 32, epi=R, resid_spatial=L.SP_UP2,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_SILU, L.SP_UP2, 1.2)]),
        Case("pnorm_1x1", [(64, 1)], 128, 1, 32, 32, epi=P,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_SILU, L.SP_SAME, 1.0)]),
        Case("cluster4_pnorm_persistent", [(256, 9)], 256, 2, 64, 64, epi=R, resid_pnorm=1,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_SAME, 1.0), (L.OUT_SILU, L.SP_SAME, 0.7)]),
        Case("cluster3_pnorm_down2", [(192, 9)], 192, 1, 32, 32, epi=R, resid_spatial=L.SP_DOWN2, resid_pnorm=1,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_DOWN2, 1.0)]),
        Case("cluster4_k1_pnorm", [(192, 1)], 256, 1, 32, 32, epi=P,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_SILU, L.SP_SAME, 1.0)]),
        Case("n128_forced_resid_pnorm", [(128, 9)], 256, 1, 32, 32, epi=R, resid_pnorm=1, n_item=128,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_SAME, 1.0)]),
        Case("n256_forced_emb", [(64, 9)], 256, 1, 32, 32, epi=E, n_item=256),
        Case("n192_forced_pnorm_2pass", [(64, 9)], 192, 1, 32, 32, epi=R, resid_pnorm=1, n_item=192,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_DOWN2, 1.0), (L.OUT_SILU, L.SP_SAME, 0.9)]),
        Case("n64_forced_c256", [(256, 9)], 256, 1, 32, 32, epi=R, n_item=64),
        Case("resident_multi_item_per_cta", [(64, 9)], 64, 3, 128, 128, epi=E),
        Case("clip_active", [(64, 9)], 64, 1, 16, 16, epi=R, clip=0.5),
        Case("clip_no_resid", [(64, 9), (64, 1)], 64, 1, 16, 16, clip=0.3),
        # ragged images: H, W multiples of 8 but not of the 16 x 8 work-item tile, several images, every spatial mode
        Case("ragged_24x40_emb", [(64, 9)], 64, 3, 24, 40, epi=E),
        Case("ragged_40x24_resid_3outs", [(128, 9)], 128, 2, 40, 24, epi=R, resid_pnorm=1,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_DOWN2, 1.0), (L.OUT_SILU, L.SP_UP2, 0.8)]),
        Case("ragged_56x72_resid_up", [(64, 9)], 64, 2, 56, 72, epi=R, resid_spatial=L.SP_UP2,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_SILU, L.SP_SAME, 1.1)]),
        Case("ragged_24x24_resid_down", [(64, 9)], 64, 2, 24, 24, epi=R, resid_spatial=L.SP_DOWN2, resid_pnorm=1,
             outs=[(L.OUT_RAW, L.SP_SAME, 1.0), (L.OUT_PNORM_SILU, L.SP_SAME, 1.0)]),
    ]
