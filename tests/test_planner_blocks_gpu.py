"""The launch planner block by block: every U-Net / autoencoder block of a planned forward against the oracle's own
block math (oracle.unet.unet_block) in fp64, fed with the GPU's stored input of that block.

One forward runs through the public call (EDMUnet2D.__call__, EDMAutoencoder.preencode / decode) on 3 images with
different noise labels and conditional inputs, at 64 x 128 so that height and width cannot be swapped unnoticed.  The
plan's arena keeps every block's bf16 `.raw` output and its side outputs, so each block is checked from what the GPU
stored as its input (for a decoder concat block: plus the encoder output the oracle's skip order names), and an error
fails at the block that makes it instead of being diluted in a whole-model comparison.

  block output   rel-RMS and max-abs error vs fp64 <= 1.25 x those of the same oracle block run under bf16 autocast
                 on the same input (DESIGN section 2, per block), its result stored in bf16 as the GPU stores `.raw`
  side outputs   `.act` (the next block's activated input), `.skip_act`, `.inv`, recomputed from the stored `.raw`:
                 per element 2^-7 |ref| + 2^-12 rms(ref) (tests/_igemm_ref.elementwise_ratio) widened by what the bf16
                 rounding of `.raw` moves the reference (the kernel works from its fp32 accumulator), and the mean of
                 got / ref - 1 within max(1e-3, 4 standard errors) (room for the bias of the kernels' tanh.approx
                 mp_silu): a scale off by a fraction of a bf16 ulp fails
  modulation     every block's cvec rows, per image, vs the oracle's c within 2e-5 (as tests/test_direct_kernels_gpu)
  output         model_out vs the oracle's mp_conv(last .raw, out_conv, out_gain), fp32 accumulation bound

The fused solves are checked for their per-step wiring: step i reads coef[i], c_in[i] and modulation set i, whose
rows are the oracle's c at that step's label; a guided step runs the guide's forward first and combines its output.
"""
from __future__ import annotations

import math

import pytest
import torch
import torch.nn.functional as F

from oracle import unet as ounet
from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import DiffusionSolve
from terrain_diffusion_b200.layout import from_nc8hw8
from terrain_diffusion_b200.models.plan import UNetProgram
from terrain_diffusion_b200.scheduler import EDMDPMSolverMultistepScheduler
from tests._igemm_ref import report
from tests.test_planner_fold_cpu import block_kwargs, eff64, model_spec, mp_concat_weights, mp_sum_weights

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
N, H, W = 3, 64, 128
LABELS = [0.35, 0.9, 1.4]
MODELS = ["decoder", "base", "guide", "coarse", "variant", "ae_encoder", "ae_decoder"]
BLOCK_FACTOR = 1.25
MEAN_TOL = 1e-3
"""Side outputs: bound on the mean of got / ref - 1.  The kernels' mp_silu uses tanh.approx.f32 (relative error up to
2^-11, csrc/tdx_ptx.cuh), which does not average out: it biases the mean by ~2e-4 (measured on an H100)."""


@pytest.fixture(scope="module")
def margins(request):
    """Worst share of each bound; written to the terminal (also under -q) when the module is done."""
    found: dict = {}
    yield found
    lines = [f"planner blocks: worst {kind}: {v[0]:.3f} ({v[1]})" for kind, v in sorted(found.items())]
    report(request.config, lines)


def _note(margins, kind, value, where):
    if kind not in margins or value > margins[kind][0]:
        margins[kind] = (value, where)


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def nchw(t: torch.Tensor) -> torch.Tensor:
    return from_nc8hw8(t).double()


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-300))


def pixel_inv(x):
    return 1.0 / (1e-4 + x.square().mean(dim=1).sqrt())


def modulation(sd, prefix, emb):
    """UNetBlock's c (unet_block.py:129-133): mp_conv(emb, emb_linear, emb_gain) + 1, RMS-normalised per row."""
    c = ounet.mp_conv(emb, sd[prefix + "emb_linear.weight"], gain=sd[prefix + "emb_gain"]) + 1
    return c / torch.sqrt(torch.mean(c ** 2, dim=1, keepdim=True) + 1e-8)


# ------------------------------------------------------------------------------------------------ one forward
def run_forward(name):
    """(spec, program, model input [N, ci, h, w] fp32, fp64 embedding or None, model output) of one public call."""
    spec = model_spec(name, DEV)
    m = spec.model.to(DEV)
    g = torch.Generator().manual_seed(17)
    if name == "ae_encoder":
        x = torch.randn(N, 1, H, W, generator=g).to(DEV)
        means, logvars = m.preencode(x)
        plans, emb, out = m.encoder._plans, None, torch.cat([means, logvars], dim=1)
    elif name == "ae_decoder":
        x = torch.randn(N, 4, H // 8, W // 8, generator=g).to(DEV)
        out = m.decode(x)
        plans, emb = m._plans, None
    else:
        cfg = spec.cfg
        x = torch.randn(N, cfg["in_channels"], H, W, generator=g).to(DEV)
        t = torch.tensor(LABELS, device=DEV)
        cond = [(torch.randn(N, dim, generator=g) if kind == "tensor" else torch.randn(N, generator=g)).to(DEV)
                for kind, dim, _ in cfg.get("conditional_inputs") or []]
        out = m(x, t, cond)
        plans = m._plans
        sd64 = {k: v.double() for k, v in spec.sd.items()}
        emb = ounet.compute_embeddings(sd64, cfg, t.double(), [c.double() for c in cond])
    assert len(plans) == 1
    prog = next(iter(plans.values()))[0]
    return spec, prog, x, emb, out


def side_check(got, raw, fn, what, margins):
    """got: stored side output; fn(v): its expected value as a function of the block output v, with any per-pixel
    normaliser held at the value computed from `raw` (the stored block output)."""
    ref = fn(raw)
    widen = (fn(raw * (1 + 2.0 ** -9)) - fn(raw * (1 - 2.0 ** -9))).abs() / 2
    bound = 2.0 ** -7 * ref.abs() + 2.0 ** -12 * float(ref.square().mean().sqrt()) + widen
    err = (got - ref).abs()
    assert not torch.isnan(got).any(), f"{what}: NaN"
    ratio = float((err / bound).max())
    big = ref.abs() > 0.1 * float(ref.square().mean().sqrt())
    r = got[big] / ref[big] - 1.0
    mean, se = float(r.mean()), float(r.std()) / math.sqrt(r.numel())
    _note(margins, "side-output error (x per-element bound)", ratio, what)
    _note(margins, "side-output mean deviation (x max(1e-3, 4 SE))", abs(mean) / max(MEAN_TOL, 4 * se), what)
    assert ratio <= 1.0, f"{what}: error {ratio:.2f} x the per-element bound"
    assert abs(mean) <= max(MEAN_TOL, 4 * se), f"{what}: mean got / ref - 1 = {mean:.3g} (standard error {se:.3g})"


def block_check(got, ref, bf, what, margins, lines, extra_abs=0.0):
    """got (GPU .raw), ref (fp64 oracle), bf (oracle under bf16 autocast, stored in bf16): rel-RMS and max-abs.
    extra_abs widens the max-abs bound by an intermediate rounding the GPU makes and the autocast block does not."""
    bf = bf.bfloat16().double()
    e, e_bf = rel_rms(got, ref), rel_rms(bf, ref)
    m, m_bf = float((got - ref).abs().max()), float((bf - ref).abs().max())
    share, share_max = e / (BLOCK_FACTOR * e_bf), m / (BLOCK_FACTOR * m_bf + extra_abs)
    lines.append(f"{what:40s} rel-RMS {e:.3e} (bf16 ref {e_bf:.3e}) share {share:.3f}; max-abs share {share_max:.3f}")
    _note(margins, "block rel-RMS share", share, what)
    _note(margins, "block max-abs share", share_max, what)
    return share, share_max


@pytest.mark.parametrize("name", MODELS)
def test_every_block_matches_the_oracle_block_from_its_stored_input(name, margins):
    spec, prog, x, emb, out = run_forward(name)
    arena, cvecs = prog.arena, prog.cvecs
    sd32 = spec.sd
    sd64 = {k: v.double() for k, v in sd32.items()}
    cfg = spec.cfg
    kw = block_kwargs(cfg)
    cb = float(cfg.get("concat_balance", 0.3))
    emb32 = emb.float() if emb is not None else None
    lines, shares = [], []

    # the first convolution over [x, ones]
    first = "enc.conv." if name == "ae_decoder" else f"enc.{spec.enc[0]['name']}."
    x0 = torch.cat([x, torch.ones_like(x[:, :1])], dim=1)
    raws = {first: nchw(arena[first + ".raw"])}
    ref = ounet.mp_conv(x0.double(), sd64[spec.first])
    with torch.autocast("cuda", dtype=torch.bfloat16):
        bf = ounet.mp_conv(x0, sd32[spec.first])
    shares.append((block_check(raws[first], ref, bf, first, margins, lines), first))

    # which decoder block takes which encoder output (oracle.unet.unet_forward: pushed per encoder stage, popped per
    # concat block), and the skip scale it applies
    seq = [(first, None, dict(spec.enc[0] if spec.enc else {}, cout=raws[first].shape[1]))] + list(spec.blocks)
    skips = [k for k, _, b in seq if k.startswith("enc.")] if spec.dec and spec.enc else []
    consumer = {}
    order = list(skips)
    for key, _, b in seq:
        if b.get("concat"):
            consumer[order.pop()] = (key, b)

    for i, (key, p, b) in enumerate(seq):
        if i > 0:
            xin = raws[seq[i - 1][0]]
            if b.get("concat"):
                xin = ounet.mp_concat([xin, raws[skips.pop()]], cb)
            ref = ounet.unet_block(xin, emb, sd64, p, b, **kw)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                bf = ounet.unet_block(xin.float(), emb32, sd32, p, b, **kw)
            raws[key] = nchw(arena[key + ".raw"])
            assert raws[key].shape == ref.shape, (key, tuple(raws[key].shape), tuple(ref.shape))
            extra = 0.0
            if key + "x1" in arena:
                # an attention block keeps x1 = mp_sum(x, y) in bf16 between its two halves and adds it back with
                # weight (1 - t) / |(1 - t, t)|: one more rounding than the autocast block, at most 2^-9 |x1| each
                extra = 2.0 ** -9 * mp_sum_weights(kw["attn_balance"])[0] * float(nchw(arena[key + "x1"]).abs().max())
            shares.append((block_check(raws[key], ref, bf, key, margins, lines, extra), key))
            # modulation vectors: rows per image
            got_c = cvecs[key].double()
            want_c = modulation(sd64, p, emb) if (p + "emb_linear.weight") in sd64 else torch.ones_like(got_c)
            err_c = float((got_c - want_c).abs().max())
            _note(margins, "cvec abs error (x 2e-5)", err_c / 2e-5, key)
            assert err_c <= 2e-5, (key, err_c)
        raw = raws[key]
        c = raw.shape[1]
        nxt = seq[i + 1][2] if i + 1 < len(seq) else None
        # the next block's activated input
        act = None
        if nxt is not None and nxt["mode"] == "enc" and nxt["cin"] == nxt["cout"]:
            inv = pixel_inv(raw)[:, None]
            act = lambda v, inv=inv, rs=nxt["resample"]: ounet.mp_silu(ounet.resample(v * inv, rs))   # noqa: E731
            got_inv = arena[key + ".inv"].double()
            err = float(((got_inv - inv[:, 0]).abs() / ((2.0 ** -9 + 2.0 ** -12) * inv[:, 0])).max())
            _note(margins, "side-output error (x per-element bound)", err, key + ".inv")
            assert err <= 1.0, (key + ".inv", err)
        elif nxt is not None and nxt["mode"] == "dec" and nxt.get("concat"):
            s1, _ = mp_concat_weights(c, nxt["skip_channels"], cb)
            act = lambda v, s1=s1: ounet.mp_silu(s1 * v)      # noqa: E731
        elif nxt is not None and nxt["mode"] == "dec":
            act = lambda v, rs=nxt["resample"]: ounet.mp_silu(ounet.resample(v, rs))   # noqa: E731
        assert (key + ".act" in arena) == (act is not None), key
        if act is not None:
            side_check(nchw(arena[key + ".act"]), raw, act, key + ".act", margins)
        if key in consumer:
            dkey, d = consumer[key]
            _, s2 = mp_concat_weights(d["cin"] - d["skip_channels"], d["skip_channels"], cb)
            side_check(nchw(arena[key + ".skip_act"]), raw, lambda v, s2=s2: ounet.mp_silu(s2 * v),
                       key + ".skip_act", margins)
        else:
            assert key + ".skip_act" not in arena, key

    # the last convolution
    last = raws[seq[-1][0]]
    w_out = eff64(sd64[spec.out[0]], spec.out[1])
    ref = F.conv2d(last, w_out, padding=1)
    scale = F.conv2d(last.abs(), w_out.abs(), padding=1)
    assert out.shape == ref.shape, (tuple(out.shape), tuple(ref.shape))
    err = float(((out.double() - ref).abs() / (2.0 ** -16 * scale + 1e-30)).max())
    _note(margins, "model_out error (x 2^-16 sum|terms|)", err, name)
    print(f"\n{name}\n" + "\n".join(lines))
    assert err <= 1.0, err
    bad = [(k, s) for s, k in shares if s[0] > 1.0 or s[1] > 1.0]
    assert not bad, f"{name}: blocks over their bound (rel-RMS share, max-abs share): {bad}"


# ------------------------------------------------------------------------------------------------ fused solves
@pytest.fixture(scope="module")
def decoder_pair():
    """The decoder (seed 0) and a guide of the same shape with other weights (seed 1)."""
    main, guide = model_spec("decoder", DEV), model_spec("decoder", DEV)
    guide.sd = {k: v.to(DEV) for k, v in ounet.procedural_state_dict(guide.cfg, seed=1).items()}
    guide.model.load_state_dict(guide.sd)
    main.model.to(DEV)
    guide.model.to(DEV)
    return main, guide


def _recording(monkeypatch):
    launches = []
    add = UNetProgram.add

    def recording_add(self, kind, desc):
        launches.append((kind, type(desc).from_buffer_copy(desc)))
        add(self, kind, desc)
    monkeypatch.setattr(UNetProgram, "add", recording_add)
    return launches


def _evaluations(launches):
    """Split a solve's launch list at its im2col launches: [[(kind, desc)] per U-Net evaluation]."""
    evals = []
    for kind, d in launches:
        if kind == "im2col":
            evals.append([])
        if evals:
            evals[-1].append((kind, d))
    return evals


def test_fused_solve_reads_each_steps_coefficients_and_modulation_set(decoder_pair, monkeypatch, margins):
    spec = decoder_pair[0]
    m, n, steps = spec.model, 2, 3
    launches = _recording(monkeypatch)
    solve = DiffusionSolve(m, EDMDPMSolverMultistepScheduler(), n, 64, 64, steps)
    g = torch.Generator().manual_seed(3)
    y = solve.run((torch.randn(n, 1, 64, 64, generator=g) * 80).to(DEV), torch.randn(n, 4, 64, 64, generator=g).to(DEV))
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    prog = solve.prog
    labels = solve.labels.double()
    assert labels.shape == (steps, n) and len(set(labels[:, 0].tolist())) == steps
    evals = _evaluations(launches)
    assert len(evals) == steps and [k for k, _ in launches].count("embed") == 1
    key_of = {t.data_ptr(): k for k, t in prog.arena.items()}
    sd64 = {k: v.double() for k, v in spec.sd.items()}
    for i, ev in enumerate(evals):
        im = ev[0][1]
        assert im.src_scale[0] == solve.c_in[i:i + 1].data_ptr(), i
        od = ev[-1][1]
        assert ev[-1][0] == "conv_out" and od.sched_coef == solve.coef[i].data_ptr(), i
        assert (od.sample, od.x0_prev) == (solve.sample.data_ptr(), solve.x0_prev.data_ptr())
        emb = ounet.compute_embeddings(sd64, spec.cfg, labels[i], [])
        n_mod = 0
        for kind, d in ev:
            if kind == "igemm" and d.epi_flags & L.EPI_EMB_SILU:
                block = key_of[d.out[0].ptr][:-1]          # res0 writes the block's `h`
                cv = prog.cvecs[block]
                assert d.cvec == cv.data_ptr() + i * n * d.c_out * 4, (i, block)
                want = modulation(sd64, block, emb)
                err = float((cv[i * n:(i + 1) * n].double() - want).abs().max())
                _note(margins, "cvec abs error (x 2e-5)", err / 2e-5, f"solve step {i} {block}")
                assert err <= 2e-5, (i, block, err)
                n_mod += 1
        assert n_mod == sum(1 for _, _, b in spec.blocks), n_mod


def test_guided_solve_runs_the_guide_first_and_combines_its_output(decoder_pair, monkeypatch):
    (main, guide), n, steps = decoder_pair, 2, 3
    launches = _recording(monkeypatch)
    solve = DiffusionSolve(main.model, EDMDPMSolverMultistepScheduler(), n, 64, 64, steps, guide=guide.model,
                           guidance_scale=1.5)
    g = torch.Generator().manual_seed(4)
    y = solve.run((torch.randn(n, 1, 64, 64, generator=g) * 80).to(DEV), torch.randn(n, 4, 64, 64, generator=g).to(DEV))
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()
    evals = _evaluations(launches)
    assert len(evals) == 2 * steps and [k for k, _ in launches].count("embed") == 2
    main_h = {t.data_ptr() for k, t in solve.prog.arena.items()}
    for i in range(steps):
        ge, me = evals[2 * i], evals[2 * i + 1]
        gd, md = ge[-1][1], me[-1][1]
        # the guide's forward: its own arena, plain model_out into the solve's guide buffer, no update
        assert all(d.out[0].ptr not in main_h for k, d in ge if k == "igemm"), i
        assert gd.model_out == solve.guide_out.data_ptr() and not gd.sched_coef and not gd.guide_out, i
        # then the main forward, whose last convolution combines the guide's output and applies step i's update
        assert all(d.out[0].ptr in main_h for k, d in me if k == "igemm"), i
        assert md.guide_out == solve.guide_out.data_ptr() and md.sched_coef == solve.coef[i].data_ptr(), i
        assert ge[0][1].src_scale[0] == me[0][1].src_scale[0] == solve.c_in[i:i + 1].data_ptr(), i
    assert float(solve.coef[0, 4]) == 1.5
