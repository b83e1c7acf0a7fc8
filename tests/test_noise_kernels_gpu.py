"""The noise field and the canvas add through their C entry points (csrc/tdx_noise.cu `tdx_noise_patch`,
`tdx_noise_patches`, `tdx_tile_seed`; csrc/tdx_direct.cu `tdx_canvas_add`), with the arguments the Python wrappers
never pass.

- Noise: guarded NaN-filled outputs against oracle/rng.py (pinned to the reference's goldens, and cross-checked here
  against its pure-Python restatement at origins and tile indices beyond +-2^31), workspaces pre-filled with 0xFF and
  guarded, the status word read after both forms, and every argument check.
- Tile seeds against oracle/rng.py and against tests/golden/tile_seed_golden.npz, recorded from the reference's own
  `_tile_seed` at large indices.
- Canvas add: the float4 and the scalar path on the same inputs, bit-identical to each other and to numpy's fp32 add
  over the clipped overlap, into a guarded destination.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import rng as orng
from terrain_diffusion_b200 import _lib as L
from tests._igemm_ref import Guarded
from tests.test_hydro_kernels_gpu import GUARD, SENTINEL, assert_bits

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
G = np.load(Path(__file__).resolve().parent / "golden" / "tile_seed_golden.npz")


class Workspace:
    """A noise workspace of `nbytes` pre-filled with 0xFF between sentinel guards."""

    def __init__(self, nbytes):
        self.nbytes = nbytes
        self.raw = torch.full((2 * GUARD + nbytes,), SENTINEL, dtype=torch.uint8, device=DEV)
        self.raw[GUARD:GUARD + nbytes].fill_(0xFF)

    def data_ptr(self):
        return self.raw[GUARD:].data_ptr()

    def check(self):
        bad = int((self.raw[:GUARD] != SENTINEL).sum()) + int((self.raw[GUARD + self.nbytes:] != SENTINEL).sum())
        assert bad == 0, f"workspace: {bad} bytes written outside it"


def run_patch(seed, y0, x0, h, w, c, th, tw):
    lib = L.lib()
    out = Guarded((c, h, w), torch.float32, DEV)
    ws = Workspace(lib.tdx_noise_patch_workspace_bytes(c, th, tw))
    L.call(lib.tdx_noise_patch, DEV, seed, y0, x0, h, w, c, th, tw, out.data_ptr(), ws.data_ptr(), ws.nbytes)
    L.call(lib.tdx_noise_patch_status, DEV, ws.data_ptr())
    out.check("noise patch")
    ws.check()
    return out.view.cpu().numpy()


def run_patches(seed, origins, h, w, c, th, tw):
    lib = L.lib()
    n = len(origins)
    out = Guarded((n, c, h, w), torch.float32, DEV)
    ws = Workspace(lib.tdx_noise_patches_workspace_bytes(c, th, tw))
    ys = (C.c_int64 * n)(*[o[0] for o in origins])
    xs = (C.c_int64 * n)(*[o[1] for o in origins])
    L.call(lib.tdx_noise_patches, DEV, seed, n, ys, xs, h, w, c, th, tw, out.data_ptr(), ws.data_ptr(), ws.nbytes)
    L.call(lib.tdx_noise_patch_status, DEV, ws.data_ptr())      # the batched form keeps its status in the same word
    out.check("noise patches")
    ws.check()
    return out.view.cpu().numpy()


NOISE_CASES = {
    # name: (base seed, origins, h, w, channels, tile_h, tile_w)
    "inside_one_tile": (5, [(5, 7), (-30, -3)], 10, 12, 1, 32, 32),
    "exactly_one_tile": (6, [(64, -32), (0, 0)], 32, 32, 2, 32, 32),
    "3x3_tiles_odd_stream": (7, [(-5, 4), (13, -20)], 20, 20, 1, 9, 9),          # C*th*tw = 81: a dropped normal
    "1x1_tiles": (8, [(3, -4), (-7, 11)], 5, 6, 3, 1, 1),                     # 30 tiles per patch, odd streams
    "six_channels": (2 ** 63 + 9, [(-20, 30), (100, -77)], 40, 20, 6, 16, 24),
    "origins_past_2_31": (9, [(2 ** 31 + 5, -2 ** 31 - 17), (-2 ** 33 - 1, 2 ** 32 + 60)], 9, 70, 1, 64, 64),
    "tile_indices_past_2_31": (2 ** 64 - 1, [(5 * 2 ** 32 + 3, -3 * 2 ** 32 - 2), (2 ** 32 - 1, -2 ** 31 - 1)],
                               4, 5, 1, 1, 1),
}


@pytest.mark.parametrize("name", list(NOISE_CASES))
def test_noise_patch_and_patches_match_the_oracle(name):
    seed, origins, h, w, c, th, tw = NOISE_CASES[name]
    batched = run_patches(seed, origins, h, w, c, th, tw)
    for i, (y0, x0) in enumerate(origins):
        want = orng.gaussian_noise_patch(seed, y0, x0, h, w, c, th, tw)
        assert_bits(run_patch(seed, y0, x0, h, w, c, th, tw), want, (name, i))
        assert_bits(batched[i], want, (name, i, "batched"))


def test_oracle_at_tile_indices_past_2_31_matches_the_python_restatement():
    seed, origins, h, w, c, _, _ = NOISE_CASES["tile_indices_past_2_31"]
    for y0, x0 in origins:
        want = np.array([[[orng.py_standard_normal(orng.py_tile_seed(seed, y0 + i, x0 + j), c)[ch] for j in range(w)]
                          for i in range(h)] for ch in range(c)], F32)
        assert np.array_equal(orng.gaussian_noise_patch(seed, y0, x0, h, w, c, 1, 1), want)


def test_noise_patches_many_jobs_share_one_counts_buffer():
    # 4 patches x 12 tiles = 48 jobs: two launches of the 32-job batch, each reusing the counts slices
    seed, origins = 21, [(0, 0), (-16, 40), (7, -9), (300, 3)]
    got = run_patches(seed, origins, 20, 30, 2, 8, 8)
    for i, (y0, x0) in enumerate(origins):
        assert_bits(got[i], orng.gaussian_noise_patch(seed, y0, x0, 20, 30, 2, 8, 8), i)


def test_tile_seed_at_large_indices():
    lib = L.lib()
    for base, (ty, tx), want in zip(G["tile_seed_large.base"].tolist(), G["tile_seed_large.args"].tolist(),
                                    G["tile_seed_large.out"].tolist()):
        assert lib.tdx_tile_seed(base, ty, tx) == want == orng.py_tile_seed(base, ty, tx) == orng.tile_seed(base, ty, tx)
    assert lib.tdx_tile_seed(3, 2 ** 32 + 5, -1) == lib.tdx_tile_seed(3, 5, 2 ** 32 - 1)   # indices mask to 32 bits


def test_noise_argument_checks():
    lib = L.lib()
    c, th, tw, h, w = 2, 16, 16, 8, 8
    need = lib.tdx_noise_patch_workspace_bytes(c, th, tw)
    need_b = lib.tdx_noise_patches_workspace_bytes(c, th, tw)
    out = Guarded((c, h, w), torch.float32, DEV)
    ws = Workspace(max(need, need_b))
    ys, xs = (C.c_int64 * 1)(0), (C.c_int64 * 1)(0)
    o, wp = out.data_ptr(), ws.data_ptr()
    single = [(None, wp, need, h, w, c, th, tw), (o, None, need, h, w, c, th, tw), (o, wp, need - 1, h, w, c, th, tw)]
    single += [(o, wp, need, *dims) for dims in ((0, w, c, th, tw), (h, 0, c, th, tw), (h, w, 0, th, tw),
                                                   (h, w, c, 0, tw), (h, w, c, th, 0), (-1, w, c, th, tw))]
    for op, wsp, nb, hh, ww, cc, tth, ttw in single:
        with pytest.raises(L.TdxError):
            L.call(lib.tdx_noise_patch, DEV, 1, 0, 0, hh, ww, cc, tth, ttw, op, wsp, nb)
    batched = [(1, ys, xs, o, wp, need_b - 1), (0, ys, xs, o, wp, need_b), (-1, ys, xs, o, wp, need_b),
               (1, None, xs, o, wp, need_b), (1, ys, None, o, wp, need_b), (1, ys, xs, None, wp, need_b),
               (1, ys, xs, o, None, need_b)]
    for n, y, x, op, wsp, nb in batched:
        with pytest.raises(L.TdxError):
            L.call(lib.tdx_noise_patches, DEV, 1, n, y, x, h, w, c, th, tw, op, wsp, nb)
    torch.cuda.synchronize()
    out.check("noise")
    ws.check()
    assert bool(torch.isnan(out.view).all()) and bool((ws.raw[GUARD:GUARD + ws.nbytes] == 0xFF).all())


def test_noise_tile_stream_of_2_30_values_is_refused():
    lib = L.lib()
    th = tw = 1 << 15                                          # C * th * tw = 2^30
    need = lib.tdx_noise_patch_workspace_bytes(1, th, tw)
    assert need > 300 << 20                                    # the full, real workspace
    ws = torch.full((need,), 0xFF, dtype=torch.uint8, device=DEV)
    out = Guarded((1, 4, 4), torch.float32, DEV)
    with pytest.raises(L.TdxError, match="too long"):
        L.call(lib.tdx_noise_patch, DEV, 1, 0, 0, 4, 4, 1, th, tw, out.data_ptr(), ws.data_ptr(), need)
    torch.cuda.synchronize()
    out.check("noise")
    assert bool(torch.isnan(out.view).all()) and bool((ws == 0xFF).all())


# ---------------------------------------------------------------------------------------------------------------------
# tdx_canvas_add
# ---------------------------------------------------------------------------------------------------------------------
def canvas_reference(dst, tile, y0, x0):
    out = dst.copy()
    _, dh, dw = dst.shape
    _, th, tw = tile.shape
    ya, yb, xa, xb = max(y0, 0), min(y0 + th, dh), max(x0, 0), min(x0 + tw, dw)
    if ya < yb and xa < xb:
        out[:, ya:yb, xa:xb] = out[:, ya:yb, xa:xb] + tile[:, ya - y0:yb - y0, xa - x0:xb - x0]
    return out


def run_canvas_add(dst, tile, y0, x0, dst_offset=0):
    """tdx_canvas_add into a guarded destination that starts `dst_offset` floats into its (16-byte aligned)
    allocation; the floats before it must stay NaN."""
    c, dh, dw = dst.shape
    _, th, tw = tile.shape
    g = Guarded((dst_offset + dst.size,), torch.float32, DEV)
    body = g.view[dst_offset:]
    body.copy_(torch.from_numpy(dst.ravel()))
    td = torch.from_numpy(np.ascontiguousarray(tile)).to(DEV)
    L.call(L.lib().tdx_canvas_add, DEV, body.data_ptr(), c, dh, dw, td.data_ptr(), th, tw, y0, x0)
    torch.cuda.synchronize()
    g.check("canvas dst")
    assert bool(torch.isnan(g.view[:dst_offset]).all())
    return body.cpu().numpy().reshape(dst.shape)


CANVAS_CASES = [
    # (channels, dst_h, dst_w, tile_h, tile_w, y0, x0)
    (1, 40, 64, 16, 32, 8, 16),          # inside
    (3, 40, 64, 16, 32, -5, -8),         # clipped top and left (negative origin)
    (3, 40, 64, 16, 32, 30, 48),         # clipped bottom and right
    (7, 20, 24, 48, 40, -12, -8),        # a tile larger than dst in both axes
    (1, 33, 36, 12, 20, 25, -4),         # bottom and left
    (7, 16, 32, 8, 16, -3, 20),          # top and right
    (3, 40, 64, 16, 32, 100, 0),         # no overlap
]


@pytest.mark.parametrize("case", CANVAS_CASES)
def test_canvas_add_vector_and_scalar_paths(case):
    c, dh, dw, th, tw, y0, x0 = case
    rng = np.random.RandomState(abs(hash(case)) % 2 ** 31)
    dst = rng.randn(c, dh, dw).astype(F32)
    tile = rng.randn(c, th, tw).astype(F32) * F32(1e3)
    want = canvas_reference(dst, tile, y0, x0)
    vec = run_canvas_add(dst, tile, y0, x0)                    # x0, widths and pointers 16-byte aligned: float4 path
    scalar = run_canvas_add(dst, tile, y0, x0, dst_offset=1)   # a 1-float offset dst: the scalar path
    assert_bits(vec, want, "float4")
    assert scalar.tobytes() == vec.tobytes()
    # x0 % 4 != 0 and an odd tile width also take the scalar path
    assert_bits(run_canvas_add(dst, tile, y0, x0 + 1), canvas_reference(dst, tile, y0, x0 + 1), "x0 % 4")
    odd = np.ascontiguousarray(tile[:, :, :tw - 1])
    assert_bits(run_canvas_add(dst, odd, y0, x0), canvas_reference(dst, odd, y0, x0), "odd tile_w")


def test_canvas_add_argument_checks():
    dst = Guarded((2, 8, 8), torch.float32, DEV)
    tile = torch.ones(2, 4, 4, device=DEV)
    d, t = dst.data_ptr(), tile.data_ptr()
    for args in ((None, 2, 8, 8, t, 4, 4), (d, 2, 8, 8, None, 4, 4), (d, 0, 8, 8, t, 4, 4), (d, 2, 0, 8, t, 4, 4),
                 (d, 2, 8, 0, t, 4, 4), (d, 2, 8, 8, t, 0, 4), (d, 2, 8, 8, t, 4, 0), (d, -2, 8, 8, t, 4, 4)):
        with pytest.raises(L.TdxError):
            L.call(L.lib().tdx_canvas_add, DEV, *args, 0, 0)
    torch.cuda.synchronize()
    dst.check("canvas dst")
    assert bool(torch.isnan(dst.view).all())
