"""Every implicit-GEMM launch plan the package runs, replayed against the fp64 reference (tests/_igemm_ref.py).

The launch descriptors of every forward on the shape surface (tests/_igemm_surface.py: the WorldPipeline stages at
their padded batches, bench.py, the evaluation batches and the tiled samplers at every `tile_batch`) are recorded on the
host, planned with this GPU's SM count and cluster occupancy, and grouped by launch plan and epilogue signature.  The
smallest launch of each group runs through tdx_igemm_run with fresh bf16-exact inputs, guarded outputs and the
per-element bound, so an error in one layer, tile row, cluster rank or last partial round fails here at that layer
instead of being diluted in a whole-model comparison.  The PRODUCT forwards' (plan class, epilogue signature) groups
run first; every finer (plan variant, epilogue signature) group of the surface that they leave out runs after them.
HAND_CASES add the paths the surface may not reach on a given GPU.
"""
from __future__ import annotations

import collections
import textwrap

import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from tests._igemm_ref import Case, check_case, needs_norm, plan_of, plan_variant, report, variant_label
from tests._igemm_surface import (gpu_tests_selected, group_key, launches, new_groups, product_representatives,
                                  surface, surface_representatives)

pytestmark = pytest.mark.gpu

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


def pytest_generate_tests(metafunc):
    cases = {"test_product_plan_matches_fp64_reference": product_representatives,
             "test_surface_plan_matches_fp64_reference": surface_representatives}.get(metafunc.function.__name__)
    if cases is not None:
        reps = cases() if gpu_tests_selected(metafunc.config) else ()
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


def test_surface_plan_matches_fp64_reference(case, margins):
    check_case(case, torch.device("cuda:0"), margins)


@pytest.mark.parametrize("case", HAND_CASES, ids=lambda c: c.name)
def test_hand_written_plan_matches_fp64_reference(case, margins):
    check_case(case, torch.device("cuda:0"), margins)


def test_every_product_plan_class_is_covered(request, margins):
    """Every (plan variant, epilogue signature) group of the surface is replayed against fp64 by one of the two
    parametrized tests above (or here, if they have not replayed it in this session), and each path listed in
    HAND_CASES is reached.  Writes to the terminal (also under -q): forwards, launches and groups; the groups the
    hand-picked PRODUCT forwards do not reach, per first source reaching them; the groups on the overlapped kernel; the
    worst per-element error; and one line per plan variant with its launch count and the case that covers it."""
    runs = launches()
    reps = list(product_representatives()) + list(surface_representatives())
    assert runs, "no launches recorded"
    keys = {group_key(la.case, la.plan) for la in runs}
    replayed = {group_key(c, plan_of(c)) for c in reps}
    assert keys <= replayed, sorted(map(str, keys - replayed))
    for c in reps:
        if c.name not in margins:
            check_case(c, torch.device("cuda:0"), margins)

    new = new_groups()
    first = collections.Counter(sources[0] for sources in new.values())
    ov = [k for k in keys if k[0][-1]]
    worst = max((c.name for c in reps), key=margins.get)
    lines = [f"igemm surface: {len(surface())} forwards, {len(runs)} launches, {len(keys)} (plan variant, epilogue) "
             f"groups, every one replayed against fp64 by {len(reps)} cases; {len(HAND_CASES)} hand-written cases",
             f"  {len(new)} groups no PRODUCT forward reaches, by the first source that does (WorldPipeline, bench, "
             f"evaluation, tiled samplers):"]
    order = [s for sources in surface().values() for s in sources]
    lines += textwrap.wrap(" ".join(f"{s}={first[s]}" for s in sorted(first, key=order.index)), 116,
                           initial_indent="    ", subsequent_indent="    ")
    lines += [f"  {len(ov)} groups run the overlapped-epilogue kernel, {sum(1 for k in ov if k in new)} of them new",
              f"  worst per-element error over the groups: {margins[worst]:.3f} of the bound ({worst})"]

    run = [(c, plan_of(c)) for c in reps + HAND_CASES]
    covered = {}
    for c, p in run:
        covered.setdefault(plan_variant(p), c.name)
    per_variant = collections.Counter(plan_variant(la.plan) for la in runs)
    lines += [f"  {variant_label(v):48s} launches={count:5d}  covered by {covered.get(v, 'NOTHING')}"
              for v, count in sorted(per_variant.items())]
    report(request.config, lines)
    assert set(per_variant) <= set(covered), sorted(set(per_variant) - set(covered))

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
    three_seg_n = {la.plan["N"] for la in runs if len(la.case.segs) == 3}
    missing += [f"3-segment concat at N = {n}" for n in sorted(three_seg_n)
                if not has(lambda c, p: len(c.segs) == 3 and p["N"] == n)]
    assert not missing, missing
