"""The implicit-GEMM shape surface (tests/_igemm_surface.py) without a GPU: it holds every batch the package's defaults
and samplers launch, derived here again from the code that launches them, and every forward on it records.

Changing a default that decides a launched batch (WorldPipeline's `latents_batch_size` or `decoder_tile_size`) must
change the surface or fail here, so the fp64 replay (tests/test_igemm_plans_gpu.py) and the overlapped-against-serial
comparison (tests/test_igemm_overlap_gpu.py) keep covering what the package runs.
"""
from __future__ import annotations

import inspect

import pytest

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference.pipeline import WorldPipeline
from terrain_diffusion_b200.inference.stages import COARSE_TILE, LATENT_TILE
from terrain_diffusion_b200.inference.tiling import padded_batch_size
from tests._igemm_ref import case_from_desc
from tests._igemm_surface import PRODUCT, Forward, record, surface


def _forwards() -> set:
    return set(surface())


@pytest.fixture()
def no_lib(monkeypatch):
    """Loading libtdx fails the test: the surface is derived from the Python defaults alone."""
    def boom(*_a, **_k):
        raise AssertionError("the surface is derived without loading libtdx")
    monkeypatch.setattr(L, "lib", boom)


def test_surface_holds_every_padded_latent_batch_of_the_default_pipeline(no_lib):
    params = inspect.signature(WorldPipeline.__init__).parameters
    sizes = params["latents_batch_size"].default
    sizes = [sizes] if isinstance(sizes, int) else list(sizes)
    padded = {padded_batch_size(n, max(sizes)) for n in range(1, max(sizes) + 1)}
    want = {f"world_latent_b{m}": Forward("base", m, LATENT_TILE) for m in padded | set(sizes)}
    want["world_decoder_b1"] = Forward("decoder", 1, params["decoder_tile_size"].default)
    want["world_coarse_b1"] = Forward("coarse", 1, COARSE_TILE)
    got = {s: f for f, sources in surface().items() for s in sources
           if s.startswith("world_latent_") or s in ("world_decoder_b1", "world_coarse_b1")}
    assert got == want


@pytest.mark.parametrize("model,hw,top", [
    ("decoder", 256, 16), ("decoder", 512, 16), ("base", LATENT_TILE, 40), ("guide", LATENT_TILE, 40),
    ("coarse", COARSE_TILE, 16), ("ae_encoder", 512, 8), ("ae_decoder", 64, 8)])
def test_surface_holds_every_sampler_tile_batch(no_lib, model, hw, top):
    want = {Forward(model, n, hw) for n in range(1, top + 1)}
    assert want <= _forwards(), sorted(want - _forwards())


def test_surface_holds_the_bench_evaluation_and_product_forwards(no_lib):
    want = {Forward("decoder", 1, 256), Forward("decoder", 16, 256), Forward("base", 40, 64),
            Forward("guide", 40, 64)}
    want |= {Forward(m, n, hw) for _, m, n, hw in PRODUCT}
    assert want <= _forwards(), sorted(want - _forwards())
    sources = [s for ss in surface().values() for s in ss]
    assert len(sources) == len(set(sources)), "one source name on two forwards"


def test_every_surface_forward_records_without_a_gpu():
    """Each forward emits igemm launches of its own batch whose descriptors replay as Cases (the library is used only
    for its host-side work-item choice)."""
    for f in surface():
        launches = record(f).igemm()
        assert launches, f
        for d in launches:
            c = case_from_desc(d)
            assert c.n == f.n and c.cout % c.n_item == 0 and c.macs > 0, (f, c)
