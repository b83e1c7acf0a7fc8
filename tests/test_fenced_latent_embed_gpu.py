"""tdx_latent_embed behind fences and behind the PDL interposer: it reads only inside its inputs, writes nothing else,
and waits for its predecessor.

This module registers the fenced cases of tdx_latent_embed with tests/test_input_extents_gpu.py (and so with
tests/test_pdl_order_gpu.py) and its fenced arguments in tests/_fence.FENCED_ARGS.  Its name sorts before
test_input_extents_*.py so that it is collected before them, and it imports without a GPU, so the coverage checks of a
CPU-only run see the new entry point too.  The kernel's values are tested in tests/test_latent_invariant_gpu.py."""
from __future__ import annotations

import pytest

from tests import test_input_extents_gpu as IE
from tests import test_pdl_order_gpu as PO
from tests._fence import FENCED_ARGS

pytestmark = pytest.mark.gpu

FENCED_ARGS["tdx_latent_embed"] = ("coarse", "cond_means", "cond_stds", "tail", "concat_scale", "noise_freqs",
                                   "noise_weight", "cond_weight")
NEW_CASES_FROM = len(IE.CASES)


@IE.case("tdx_latent_embed", (1, 6, 192, 768), (3, 1, 4, 20), (5, 6, 16, 300))
def _latent_embed(env, n, n_tail, noise_dims, emb):
    d = 52 + n_tail
    win = IE._rand(90 + n, n, 7, 16, lo=-2.0, hi=2.0)
    win[:, 6] = abs(win[:, 6]) + 0.25                              # the weight channel: no zero weights here
    coarse = env.inp("coarse", win)
    means = env.inp("cond_means", IE._rand(91, 7, lo=-1.0, hi=1.0))
    stds = env.inp("cond_stds", IE._rand(92, 7, lo=0.5, hi=2.0))
    tail = env.inp("tail", IE._rand(93, n_tail))
    scale = env.inp("concat_scale", IE._rand(94, d, lo=0.2, hi=1.5))
    freqs = env.inp("noise_freqs", IE._rand(95, noise_dims // 2, lo=0.0, hi=1.0))
    wn = env.inp("noise_weight", IE._rand(96, noise_dims, emb, lo=-0.1, hi=0.1))
    wc = env.inp("cond_weight", IE._rand(97, d, emb, lo=-0.1, hi=0.1))
    out = env.out("emb", (n, emb))
    vec = env.out("cond_vec", (n, d))
    IE.call("tdx_latent_embed", out.data_ptr(), vec.data_ptr(), coarse.data_ptr(), means.data_ptr(), stds.data_ptr(),
            tail.data_ptr(), n_tail, scale.data_ptr(), freqs.data_ptr(), wn.data_ptr(), wc.data_ptr(), noise_dims, emb,
            1.25, 1.0, 0.5, 1.118034, n)


NEW_CASES = IE.CASES[NEW_CASES_FROM:]


@pytest.mark.parametrize("c", NEW_CASES, ids=[c.name for c in NEW_CASES])
def test_latent_embed_reads_only_inside_its_inputs(c):
    IE.run_case(c)


@pytest.mark.parametrize("c", NEW_CASES, ids=[c.name for c in NEW_CASES])
def test_latent_embed_waits_for_its_predecessor(c):
    PO.run_interposed(c)


def test_cases_are_registered():
    assert [c.entry for c in NEW_CASES] == ["tdx_latent_embed"] * 3
