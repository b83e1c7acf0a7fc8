"""Host-side contract of the program API and of the packed-weight size (no GPU needed): the argument checks of
tdx_program_* return before any CUDA call, and tdx_igemm_packed_weight_elems sizes the B operand of every segment
configuration the shipped models launch exactly as layout.pack_weight_segments packs it."""
from __future__ import annotations

import ctypes as C

import torch

from terrain_diffusion_b200 import _lib as L
from terrain_diffusion_b200.layout import pack_weight_segments
from tests._capture import CONFIGS, capture_forward

ADDS = [("tdx_program_add_im2col", L.TdxIm2colDesc), ("tdx_program_add_igemm", L.TdxIgemmDesc),
        ("tdx_program_add_conv_out", L.TdxConvOutDesc), ("tdx_program_add_embed", L.TdxEmbedDesc),
        ("tdx_program_add_attn", L.TdxAttnDesc)]


def _invalid(rc, what):
    assert rc == -1, (what, rc)                                     # TDX_E_INVALID
    msg = L.lib().tdx_last_error().decode()
    assert "program" in msg and "null" in msg, (what, msg)


def test_program_entry_points_refuse_null_arguments():
    lib = L.lib()
    _invalid(lib.tdx_program_create(None), "create")
    _invalid(lib.tdx_program_run(None, 1, None), "run")
    _invalid(lib.tdx_program_run(None, 0, None), "run eager")
    _invalid(lib.tdx_program_instantiate(None, None), "instantiate")
    ms, kinds = (C.c_float * 1)(), (C.c_int32 * 1)()
    _invalid(lib.tdx_program_profile(None, ms, kinds, None), "profile")
    assert lib.tdx_program_num_launches(None) == -1
    assert lib.tdx_program_destroy(None) == 0
    h = C.c_void_p()
    assert lib.tdx_program_create(C.byref(h)) == 0 and h.value
    try:
        assert lib.tdx_program_num_launches(h) == 0
        _invalid(lib.tdx_program_profile(h, None, kinds, None), "profile without a time buffer")
        for name, desc in ADDS:
            _invalid(getattr(lib, name)(None, C.byref(desc())), f"{name} without a program")
            _invalid(getattr(lib, name)(h, None), f"{name} without a descriptor")
        assert lib.tdx_program_num_launches(h) == 0
    finally:
        assert lib.tdx_program_destroy(h) == 0


def _product_segments():
    """Every distinct (segments [(channels, taps)], c_out, n_per_item) of the igemm launches the shipped models record."""
    found = set()
    for name, n, hw in (("decoder", 1, 64), ("base", 1, 64), ("guide", 1, 64), ("coarse", 1, 16)):
        assert name in CONFIGS
        for d in capture_forward(name, n, hw).igemm():
            segs = tuple((int(d.a_channels[i]), int(d.a_taps[i])) for i in range(d.n_seg))
            found.add((segs, int(d.c_out), int(d.n_per_item)))
    return sorted(found)


def test_packed_weight_elems_matches_the_packing():
    configs = _product_segments()
    assert any(len(s) == 3 for s, _, _ in configs) and any(t == 1 for s, _, _ in configs for _, t in s)
    for segs, c_out, n_item in configs:
        ch = (C.c_int32 * 3)(*[c for c, _ in segs], *([0] * (3 - len(segs))))
        tp = (C.c_int32 * 3)(*[t for _, t in segs], *([0] * (3 - len(segs))))
        got = L.lib().tdx_igemm_packed_weight_elems(ch, tp, len(segs), c_out)
        ws = [torch.zeros(c_out, c, 3 if t == 9 else 1, 3 if t == 9 else 1) for c, t in segs]
        assert got == pack_weight_segments(ws, n_item).numel(), (segs, c_out, n_item)
