"""Every implicit-GEMM launch plan the shipped models run, replayed against the fp64 reference (tests/_igemm_ref.py).

The launch descriptors of the product's forwards (PRODUCT) are recorded on the host (tests/_capture.py), planned with
this GPU's SM count and cluster occupancy, and grouped by (plan class, epilogue signature).  The smallest launch of
each group runs through tdx_igemm_run with fresh bf16-exact inputs, guarded outputs and the per-element bound, so an
error in one layer, tile row or cluster rank fails here at that layer instead of being diluted in a whole-model
comparison.  HAND_CASES add the paths the product may not reach on a given GPU.
"""
from __future__ import annotations

import collections
import functools

import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from tests._capture import capture_forward, layer_of
from tests._igemm_ref import (Case, case_from_desc, check_case, needs_norm, plan_class, plan_label, plan_of,
                              report)

pytestmark = pytest.mark.gpu

PRODUCT = [
    # (source, model, batch, tile size)
    ("bench_tiles1", "decoder", 1, 256),           # bench.py (decoder solve, 256^2 tiles)
    ("bench_tiles16", "decoder", 16, 256),
    ("world_decoder_b1", "decoder", 1, 512),       # WorldPipeline decoder windows of 512, batches 1-16
    ("world_decoder_b8", "decoder", 8, 512),
    ("world_decoder_b16", "decoder", 16, 512),
    ("decoder_64", "decoder", 1, 64),
    ("decoder_128_b2", "decoder", 2, 128),
    ("latent_b1", "base", 1, 64),                  # latent stage, batches 1-16 of 64^2 tiles
    ("latent_b2", "base", 2, 64),
    ("latent_b16", "base", 16, 64),
    ("guided_main_b40", "base", 40, 64),           # guided base diffusion: 40 tiles, main model and guide
    ("guide_b16", "guide", 16, 64),
    ("guided_guide_b40", "guide", 40, 64),
    ("coarse_b1", "coarse", 1, 64),
    ("coarse_b16", "coarse", 16, 64),
]

E, R, P = L.EPI_EMB_SILU, L.EPI_RESID, L.EPI_PNORM
RAW, SILU, PSILU = L.OUT_RAW, L.OUT_SILU, L.OUT_PNORM_SILU
SAME = L.SP_SAME
HAND_CASES = [
    # split-K over a cluster on a ragged 8 x 8 image (the latent model's deepest level)
    Case("hand_splitk_ragged_8x8_c768_emb", [(768, 9)], 768, 1, 8, 8, epi=E),
    # pixel-norm statistics across a cluster of 8 CTAs (N = 64) on a ragged 8 x 8 image, side planes in and out
    Case("hand_pnorm_cluster8_ragged_8x8_c512", [(512, 9)], 512, 1, 8, 8, epi=R, resid_pnorm=1, resid_inv=True,
         n_item=64, clip=256.0, outs=[(RAW, SAME, 1.0), (PSILU, SAME, 1.0)], rms_out=True),
    # pixel-norm statistics across a 4-CTA cluster, 4 rounds per CTA, last round partial (x_full parity alternates)
    Case("hand_pnorm_cluster4_multiround", [(256, 9)], 512, 4, 64, 64, epi=R, resid_pnorm=1, n_item=128,
         outs=[(RAW, SAME, 1.0), (PSILU, SAME, 1.0), (SILU, SAME, 0.8)], rms_out=True),
    # weights streamed through the ring, several rounds per CTA
    Case("hand_stream_multiround", [(256, 9)], 128, 16, 64, 64, epi=E, n_item=128),
    # resident weights, several rounds per CTA
    Case("hand_resident_multiround", [(64, 9)], 64, 3, 128, 128, epi=E),
    # the widest work item: a one-slot weight ring
    Case("hand_n256_stream", [(256, 9)], 256, 2, 64, 64, epi=R, n_item=256, outs=[(RAW, SAME, 1.0), (SILU, SAME, 0.9)]),
    Case("hand_n256_pnorm_ragged", [(128, 9), (64, 1)], 256, 2, 24, 40, epi=P, n_item=256,
         outs=[(RAW, SAME, 1.0), (SILU, SAME, 1.0)]),
]


def epilogue_signature(c: Case) -> tuple:
    """Epilogue flags, residual mode, pixel-norm side planes, outputs (kind, spatial), clip on/off, tap pattern."""
    has_resid = bool(c.epi & R)
    return (c.epi, c.resid_spatial if has_resid else None, c.resid_pnorm if has_resid else None, c.resid_inv,
            c.rms_out, tuple((k, s) for k, s, _ in c.outs), c.clip > 0, tuple(t for _, t in c.segs))


def _signature_label(sig) -> str:
    epi, rsp, rpn, rinv, rms, outs, clip, taps = sig
    parts = ["e" + str(epi)]
    if rsp is not None:
        parts.append(f"r{rsp}{'inv' if rinv else ('pn' if rpn else '')}")
    if rms:
        parts.append("rms")
    parts.append("o" + "".join(f"{k}{s}" for k, s in outs))
    if clip:
        parts.append("clip")
    parts.append("t" + "".join(str(t) for t in taps))
    return ".".join(parts)


def product_launches() -> list:
    """[(source, layer, case, plan)] for every igemm launch of PRODUCT, planned on this device."""
    out = []
    for source, model, n, hw in PRODUCT:
        prog = capture_forward(model, n, hw)
        for d in prog.igemm():
            c = case_from_desc(d, name=f"{source}:{layer_of(prog, d)}")
            out.append((source, layer_of(prog, d), c, plan_of(c)))
    return out


def representatives(launches) -> list:
    """The smallest launch (fewest MACs) of every (plan class, epilogue signature) group, as a named Case."""
    groups: dict = {}
    for source, layer, c, p in launches:
        key = (plan_class(p), epilogue_signature(c))
        if key not in groups or c.macs < groups[key][0].macs:
            groups[key] = (c, p)
    reps = []
    for (cls, sig), (c, p) in sorted(groups.items(), key=lambda kv: (kv[0][0], str(kv[0][1]))):
        c.name = f"{plan_label(cls)}-{_signature_label(sig)}-{c.name}"
        reps.append(c)
    return reps


@functools.lru_cache(maxsize=None)
def product() -> tuple:
    """(launches, representatives) of PRODUCT on this GPU, recorded once per session."""
    launches = product_launches()
    return launches, representatives(launches)


def _gpu_tests_selected(config) -> bool:
    """Whether this run executes gpu-marked tests: only then is the product recorded (it folds four models)."""
    if not torch.cuda.is_available():
        return False
    expr = config.getoption("markexpr")
    if not expr:
        return True
    try:
        from _pytest.mark.expression import Expression
        return bool(Expression.compile(expr).evaluate(lambda name, **kw: name == "gpu"))
    except Exception:
        return True


def pytest_generate_tests(metafunc):
    if metafunc.function.__name__ == "test_product_plan_matches_fp64_reference":
        reps = product()[1] if _gpu_tests_selected(metafunc.config) else []
        metafunc.parametrize("case", reps, ids=lambda c: c.name)


@pytest.fixture(scope="module")
def margins(request):
    """Worst per-element error per case; the worst one is written to the terminal when the module is done."""
    found: dict = {}
    yield found
    if found:
        worst = max(found, key=found.get)
        report(request.config, [f"igemm: worst per-element error {found[worst]:.3f} of the bound ({worst})"])


def test_product_plan_matches_fp64_reference(case, margins):
    check_case(case, torch.device("cuda:0"), margins)


@pytest.mark.parametrize("case", HAND_CASES, ids=lambda c: c.name)
def test_hand_written_plan_matches_fp64_reference(case, margins):
    check_case(case, torch.device("cuda:0"), margins)


def test_every_product_plan_class_is_covered(request):
    """Every plan class the product reaches on this GPU is replayed above, and so is each path listed in HAND_CASES.
    Writes one line per class to the terminal (also under -q): launches in PRODUCT and the case that covers it."""
    launches, reps = product()
    assert launches, "no product launches recorded"
    run = [(c, plan_of(c)) for c in reps + HAND_CASES]
    covered = {}
    for c, p in run:
        covered.setdefault(plan_class(p), c.name)
    per_class = collections.Counter(plan_class(p) for _, _, _, p in launches)
    lines = [f"{len(per_class)} product plan classes, {len(launches)} launches, {len(reps)} groups replayed, "
             f"{len(HAND_CASES)} hand-written cases"]
    lines += [f"  {plan_label(cls):32s} launches={count:4d}  covered by {covered.get(cls, 'NOTHING')}"
              for cls, count in sorted(per_class.items())]
    report(request.config, lines)
    assert set(per_class) <= set(covered), sorted(set(per_class) - set(covered))

    def has(pred):
        return any(pred(c, p) for c, p in run)

    missing = [name for name, pred in [
        ("split-K ks >= 4 on a ragged image", lambda c, p: p["ks"] >= 4 and p["ragged"]),
        ("pixel-norm cluster, >= 3 rounds, partial last round",
         lambda c, p: needs_norm(c) and p["cluster"] > 1 and p["ks"] == 1 and p["rounds"] >= 3 and p["partial"]),
        ("streaming ring, >= 3 rounds", lambda c, p: not p["resident"] and p["rounds"] >= 3),
        ("resident ring, >= 3 rounds", lambda c, p: p["resident"] and p["rounds"] >= 3),
        ("SB = 1", lambda c, p: not p["resident"] and p["SB"] == 1),
        ("N = 256", lambda c, p: p["N"] == 256),
    ] if not has(pred)]
    three_seg_n = {p["N"] for _, _, c, p in launches if len(c.segs) == 3}
    missing += [f"3-segment concat at N = {n}" for n in sorted(three_seg_n)
                if not has(lambda c, p: len(c.segs) == 3 and p["N"] == n)]
    assert not missing, missing
