"""Host-side layout helpers: NC8HW8 activations and packed wgmma weight stages (see include/tdx.h)."""
from __future__ import annotations

import torch


def to_nc8hw8(x: torch.Tensor) -> torch.Tensor:
    """[N, C, H, W] -> bf16 [N, C/8, H, W, 8] (channel groups of 8 innermost)."""
    n, c, h, w = x.shape
    assert c % 8 == 0, c
    return x.reshape(n, c // 8, 8, h, w).permute(0, 1, 3, 4, 2).contiguous().to(torch.bfloat16)


def from_nc8hw8(t: torch.Tensor) -> torch.Tensor:
    """bf16 [N, C/8, H, W, 8] -> fp32 [N, C, H, W]."""
    n, c8, h, w, e = t.shape
    assert e == 8
    return t.permute(0, 1, 4, 2, 3).reshape(n, c8 * 8, h, w).float()


def pack_weight_segments(segments: list[torch.Tensor], n_per_item: int = 64) -> torch.Tensor:
    """Pack effective conv weights into the kernel's B-stage order.

    segments: list of fp32 [Cout, Cs, kh, kw] tensors (kh=kw=3 or 1), Cs multiple of 64, in K-loop order;
    n_per_item: output channels per work item (MMA N; 64/128/192/256, divides Cout) -- see tdx_igemm_choose_n.
    Layout: [Cout/n slices][stage = (segment, 64-channel chunk, tap r*3+c)][8 k-groups][n out channels][8 channels]
    bf16 -- every stage is the K-major no-swizzle core-matrix image the MMA reads (LBO = n*16 B between k-groups,
    SBO = 128 B between 8-row groups), and each output slice owns a contiguous stream of stages.
    """
    parts = []
    cout = segments[0].shape[0]
    n = n_per_item
    assert cout % n == 0 and n % 64 == 0, (cout, n)
    for w in segments:
        co, cs, kh, kw = w.shape
        assert co == cout and cs % 64 == 0 and (kh, kw) in ((3, 3), (1, 1))
        taps = kh * kw
        v = w.reshape(co // n, n, cs // 64, 8, 8, taps)       # [split, n, chunk, kg, e, tap]
        v = v.permute(0, 2, 5, 3, 1, 4).contiguous()          # [split, chunk, tap, kg, n, e]
        parts.append(v.reshape(co // n, -1))
    return torch.cat(parts, dim=1).reshape(-1).to(torch.bfloat16).contiguous()
