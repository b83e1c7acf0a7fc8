"""Host-side checks of the launch list and of the direct kernels' descriptor validation (no GPU needed)."""
from __future__ import annotations

import collections
import ctypes as C

import pytest

from terrain_diffusion_b200 import _lib as L
from tests._capture import capture_forward


@pytest.mark.parametrize("model,n,hw,igemm,attn", [("decoder", 1, 64, 76, 0), ("decoder", 16, 512, 76, 0),
                                                    ("base", 1, 64, 80, 1), ("base", 40, 64, 80, 1),
                                                    ("guide", 16, 64, 80, 1), ("coarse", 1, 64, 15, 0)])
def test_forward_launch_list_is_recorded_without_a_gpu(model, n, hw, igemm, attn):
    """One forward = one embed, one im2col, the igemm launches, the attention cores and one conv_out; the recorded
    descriptors carry the shape and distinct (stand-in) buffers, including the pixel-norm side planes."""
    prog = capture_forward(model, n, hw)
    kinds = collections.Counter(k for k, _ in prog.launches)
    assert kinds == collections.Counter(embed=1, im2col=1, igemm=igemm, attn=attn, conv_out=1) - collections.Counter()
    assert prog.n_igemm == igemm and prog.n_launch == len(prog.launches)
    ds = prog.igemm()
    assert all(d.n_img == n for d in ds)
    assert all(d.out[0].ptr for d in ds)
    assert any(d.rms_out for d in ds) and any(d.resid_inv for d in ds)
    assert all(not d.resid_pnorm for d in ds if d.resid_inv)
    assert ds[0].height == hw and ds[-1].height == hw


_SLOT = 512 * 1024
_ARENA = None


def _addr(i: int) -> int:
    """Address for pointer field i of a descriptor: a 512 KiB slot of one zeroed device buffer when a GPU is present
    (large enough for every descriptor below, so even a descriptor that slipped through validation would stay in
    bounds), else an arbitrary non-null value (without a device nothing can be launched)."""
    global _ARENA
    import torch
    if not torch.cuda.is_available():
        return 0x100000 * (i + 1)
    if _ARENA is None:
        _ARENA = torch.zeros(8 * _SLOT, dtype=torch.uint8, device="cuda")
    return _ARENA.data_ptr() + i * _SLOT


def _rejects(fn, desc, field):
    rc = fn(C.byref(desc), None)
    assert rc == -1, rc                                       # TDX_E_INVALID: refused before any CUDA call
    assert field in L.lib().tdx_last_error().decode()


def _conv_out_desc(**kw):
    d = L.TdxConvOutDesc()
    d.x, d.weight, d.model_out = _addr(0), _addr(1), _addr(2)
    # a 0 x 0 image (conv_out_validate does not look at the shape) gives an empty grid: no kernel could run even if a
    # check regressed, including the guided one that would read the missing coefficients
    d.c_in, d.c_out, d.n_img, d.height, d.width = 64, 1, 1, 0, 0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_conv_out_rejects_bad_descriptors():
    run = L.lib().tdx_conv_out_run
    _rejects(run, _conv_out_desc(c_in=12), "c_in")
    _rejects(run, _conv_out_desc(c_out=9), "c_out")
    _rejects(run, _conv_out_desc(guide_out=_addr(3)), "guide_out")


def _embed_desc(n_blocks=4, **kw):
    arr = (L.TdxEmbedBlock * n_blocks)()
    for b in arr:
        b.weight, b.cvec, b.c_out = _addr(0), _addr(1), 64
    d = L.TdxEmbedDesc()
    d.noise_labels, d.noise_weight, d.noise_freqs = _addr(2), _addr(3), _addr(4)
    d.noise_dims, d.emb_channels, d.n_img, d.n_blocks, d.blocks = 64, 256, 1, n_blocks, arr
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_embed_rejects_bad_descriptors():
    run = L.lib().tdx_embed_run
    _rejects(run, _embed_desc(n_blocks=65), "n_blocks")
    _rejects(run, _embed_desc(emb_channels=200), "emb_channels")
    _rejects(run, _embed_desc(noise_dims=6), "noise_dims")


def _attn_desc(**kw):
    d = L.TdxAttnDesc()
    d.q, d.k, d.v, d.out = _addr(0), _addr(1), _addr(2), _addr(3)
    d.n_img, d.heads, d.head_dim, d.tokens = 1, 12, 64, 64
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_attn_rejects_bad_descriptors():
    run = L.lib().tdx_attn_run
    _rejects(run, _attn_desc(head_dim=32), "head_dim")
    _rejects(run, _attn_desc(tokens=263), "tokens")
