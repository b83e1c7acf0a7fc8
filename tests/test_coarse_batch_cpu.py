"""The batched coarse stage without a GPU: `WorldPipeline(coarse_batch_size=)` and `coarse_stage_tiles` argument checks,
the option's absence from config.json, the batch-invariant launch plans of the coarse model (recorded on the host,
tests/_capture.py) and the ctypes declarations of the new entry points against include/tdx.h."""
import ctypes as C
import json
import re

import pytest
import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.inference import WorldPipeline
from terrain_diffusion_b200.inference.stages import COARSE_BATCH_SIZES, coarse_stage_tiles
from tests._capture import RecordingEmitter, RecordingProgram, folded
from tests.test_abi_decl_cpu import PROTOTYPES, _kind

NEW_ENTRY_POINTS = ("tdx_coarse_condition", "tdx_synthetic_maps")


# ------------------------------------------------------------------------------------------------ the option
@pytest.mark.parametrize("bad", [0, 3, 5, 32, -1, 2.0, "4", None])
def test_illegal_coarse_batch_size_raises_in_the_constructor(bad):
    with pytest.raises(ValueError, match="coarse_batch_size"):
        WorldPipeline(seed=1, coarse_batch_size=bad)


@pytest.mark.parametrize("size", COARSE_BATCH_SIZES)
def test_legal_coarse_batch_sizes(size):
    assert COARSE_BATCH_SIZES == (1, 2, 4, 8, 16)
    assert WorldPipeline(seed=1, coarse_batch_size=size).coarse_batch_size == size


def test_default_is_one_window_at_a_time():
    assert WorldPipeline(seed=1).coarse_batch_size == 1


def test_coarse_batch_size_is_kept_out_of_the_config(tmp_path):
    assert "coarse_batch_size" in WorldPipeline.ignore_for_config
    WorldPipeline(seed=1, coarse_batch_size=16).save_pretrained(tmp_path)
    cfg = json.loads((tmp_path / "config.json").read_text())
    assert "coarse_batch_size" not in cfg
    assert WorldPipeline(**cfg, seed=1).coarse_batch_size == 1


# ------------------------------------------------------------------------------------------------ coarse_stage_tiles
def _args(n_ctx, n_maps, pool=1):
    ctxs = [(0, i, -i) for i in range(n_ctx)]
    maps = [torch.zeros(5, 64, 64) for _ in range(n_maps)]
    return dict(model=None, scheduler=None, seed=0, ctxs=ctxs, synthetic_maps=maps, t_cond=torch.zeros(5),
                cond_inputs=[], weight_window=torch.ones(64 // pool, 64 // pool), coarse_means=[0.0] * 6,
                coarse_stds=[1.0] * 6, pool_size=pool)


@pytest.mark.parametrize("n_ctx,n_maps", [(2, 1), (1, 2), (0, 1), (16, 15)])
def test_mismatched_windows_and_maps_raise(n_ctx, n_maps):
    with pytest.raises(ValueError, match="conditioning maps"):
        coarse_stage_tiles(**_args(n_ctx, n_maps))


def test_more_than_sixteen_windows_raise():
    with pytest.raises(ValueError, match="at most 16"):
        coarse_stage_tiles(**_args(17, 17))


def test_illegal_pool_size_raises_before_anything_else():
    with pytest.raises(ValueError, match="coarse_pooling"):
        coarse_stage_tiles(**_args(2, 1, pool=3))


def test_no_windows_no_work():
    assert coarse_stage_tiles(**_args(0, 0)) == []


# ------------------------------------------------------------------------------------------------ launch plans
def recorded(n, batch_invariant):
    """The igemm descriptors of one coarse-model forward on n 64^2 windows, recorded on the host."""
    fw = folded("coarse")
    prog = RecordingProgram()
    em = RecordingEmitter(fw, n, 64, 64, prog)
    em.batch_invariant = batch_invariant
    meta = torch.device("meta")
    em.emit_embed(prog, emb_in=torch.empty((n, fw.emb_channels), device=meta))
    x = torch.empty((n, fw.in_channels, 64, 64), device=meta)
    em.emit(prog, [(x, fw.in_channels, None)], model_out=torch.empty((n, fw.out_channels, 64, 64), device=meta))
    return prog.igemm()


def test_batch_invariant_plans_force_the_one_image_shape():
    """Every launch of a batch-invariant forward carries the forced split-K factor of its one-image launch, with that
    launch's N, and the library reports exactly that shape at every batch size (this host's fallback occupancy: the
    GPU tests repeat it with the H100's)."""
    plain = [L.igemm_launch_shape(d) for d in recorded(1, False)]
    for n in range(1, 17):
        descs = recorded(n, True)
        assert [(int(d.n_per_item), int(d.ksplit)) for d in descs] == plain, n
        assert [L.igemm_launch_shape(d) for d in descs] == plain, n
    assert all(int(d.ksplit) == 0 for d in recorded(16, False))     # existing plans force nothing


def test_forced_ksplit_is_validated_without_a_gpu():
    d = L.TdxIgemmDesc()
    d.n_seg, d.a_ptr[0], d.a_channels[0], d.a_taps[0] = 1, 16, 128, 9
    d.b_packed, d.c_out, d.n_per_item, d.n_img, d.height, d.width = 32, 128, 64, 1, 64, 64
    d.out[0].ptr, d.out[0].kind = 48, L.OUT_RAW
    d.ksplit = 3                                   # 64 columns do not split into 3 parts of 32
    assert L.lib().tdx_igemm_run(C.byref(d), None) == -1
    assert b"forced ksplit=3" in L.lib().tdx_last_error()
    d.ksplit = 9
    with pytest.raises(L.TdxError, match="ksplit=9"):
        L.igemm_launch_shape(d)
    for ks in (1, 2):
        d.ksplit = ks
        for n in (1, 7, 16):
            d.n_img = n
            assert L.igemm_launch_shape(d) == (64, ks)


# ------------------------------------------------------------------------------------------------ declarations
def test_descriptor_has_the_forced_ksplit_field_last():
    names = [f[0] for f in L.TdxIgemmDesc._fields_]
    assert names[-2:] == ["ksplit", "_pad"]
    assert L.lib().tdx_abi_sizeof(1) == C.sizeof(L.TdxIgemmDesc)


@pytest.mark.parametrize("name", NEW_ENTRY_POINTS)
def test_new_entry_point_declarations_match_the_header(name):
    ret, args = PROTOTYPES[name]
    fn = getattr(L.lib(), name)
    assert [_kind(t) for t in fn.argtypes] == args
    assert _kind(fn.restype) == ret


def test_shape_query_declaration_matches_its_definition():
    """tdx_debug_igemm_launch_shape is a host-only query exported beside tdx_debug_igemm_plan (not part of tdx.h)."""
    from tests.test_entry_points_cpu import CSRC
    src = (CSRC / "tdx_igemm.cu").read_text()
    m = re.search(r'extern "C" int tdx_debug_igemm_launch_shape\(const TdxIgemmDesc\* desc, int32_t\* shape\)', src)
    assert m
    fn = L.lib().tdx_debug_igemm_launch_shape
    assert fn.restype is C.c_int and fn.argtypes == [C.POINTER(L.TdxIgemmDesc), C.POINTER(C.c_int32)]
