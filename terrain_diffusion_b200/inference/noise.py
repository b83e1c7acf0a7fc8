"""Deterministic tile-seeded Gaussian noise field, generated on the GPU bit-compatibly with the reference's
sequential numba generator (inference/portable_rng.py:55-82, world_pipeline.py:58-115)."""
from __future__ import annotations

import torch

from .. import _lib as L

MASK64 = 0xFFFFFFFFFFFFFFFF


def tile_seed(base_seed: int, ty: int, tx: int) -> int:
    """_tile_seed (world_pipeline.py:58-63)."""
    return int(L.lib().tdx_tile_seed(int(base_seed) & MASK64, int(ty), int(tx)))


def next_seed(seed: int | None) -> int:
    """Derive a new 64-bit seed from a parent seed, or from the clock when seed is None / 0 (portable_rng.py:31-42):
    two PCG-XSH-RR 64/32 outputs, low word first.  Host integer arithmetic (a seed is drawn once per world)."""
    state = (int(seed) & MASK64) if seed is not None else 0
    if state == 0:
        import time
        state = int(time.perf_counter_ns()) & MASK64

    def step(st):
        st = (st * 6364136223846793005 + 1442695040888963407) & MASK64
        x = (((st >> 18) ^ st) >> 27) & 0xFFFFFFFF
        rot = st >> 59
        return st, ((x >> rot) | (x << ((32 - rot) & 31))) & 0xFFFFFFFF

    state, lo = step(state)
    state, hi = step(state)
    return int(((hi << 32) | lo) & MASK64)


_workspaces: dict = {}


def gaussian_noise_patch(base_seed: int, y0: int, x0: int, h: int, w: int, channels: int = 1, tile_h: int = 256,
                         tile_w: int = 256, device="cuda", check: bool = False) -> torch.Tensor:
    """(C, h, w) fp32 CUDA tensor: the patch at integer world origin (y0, x0); negative coordinates supported."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise L.TdxError("gaussian_noise_patch (GPU path) generates on the GPU; there is no CPU path")
    nbytes = int(L.lib().tdx_noise_patch_workspace_bytes(channels, tile_h, tile_w))
    # one scratch per (device, size, stream): two streams of one device must not share the counts / status words
    key = (dev, nbytes, L.current_stream_ptr(dev))
    if key not in _workspaces:
        _workspaces[key] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    ws = _workspaces[key]
    out = torch.empty((channels, h, w), dtype=torch.float32, device=dev)
    L.call(L.lib().tdx_noise_patch, dev, int(base_seed) & MASK64, int(y0), int(x0), h, w, channels, tile_h, tile_w,
           out.data_ptr(), ws.data_ptr(), nbytes)
    if check:
        L.call(L.lib().tdx_noise_patch_status, dev, ws.data_ptr())
    return out


def gaussian_noise_patches(base_seed: int, origins, h: int, w: int, channels: int = 1, tile_h: int = 256,
                           tile_w: int = 256, device="cuda") -> torch.Tensor:
    """[n, C, h, w]: the patches at the integer world origins `origins` = [(y0, x0), ...] in ONE library call (three
    launches per 32 (patch, tile) pairs); bit-identical to stacking gaussian_noise_patch results."""
    import ctypes as C
    dev = torch.device(device)
    if dev.type != "cuda":
        raise L.TdxError("gaussian_noise_patches (GPU path) generates on the GPU; there is no CPU path")
    n = len(origins)
    out = torch.empty((n, channels, h, w), dtype=torch.float32, device=dev)
    if n == 0:
        return out
    nbytes = int(L.lib().tdx_noise_patches_workspace_bytes(channels, tile_h, tile_w))
    key = (dev, nbytes, L.current_stream_ptr(dev))
    if key not in _workspaces:
        _workspaces[key] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    ws = _workspaces[key]
    ys = (C.c_int64 * n)(*[int(o[0]) for o in origins])
    xs = (C.c_int64 * n)(*[int(o[1]) for o in origins])
    L.call(L.lib().tdx_noise_patches, dev, int(base_seed) & MASK64, n, ys, xs, h, w, channels, tile_h, tile_w,
           out.data_ptr(), ws.data_ptr(), nbytes)
    return out


def standard_normal(seed: int, n: int, device="cuda") -> torch.Tensor:
    """portable_rng.standard_normal(seed, n) as an fp32 CUDA tensor (bit-identical stream)."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise L.TdxError("standard_normal (GPU path) generates on the GPU; there is no CPU path")
    out = torch.empty((n,), dtype=torch.float32, device=dev)
    if n == 0:
        return out
    nbytes = int(L.lib().tdx_noise_patch_workspace_bytes(1, 1, n))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    L.call(L.lib().tdx_standard_normal, dev, int(seed) & MASK64, n, out.data_ptr(), ws.data_ptr(), nbytes)
    return out
