"""The coarse tile's epilogue (world_pipeline.py:948-958, with `_pool_coarse_conditioning` / `_pool_channel` at
:994-1016) restated in torch CPU fp32 elementwise ops, with the pooling written out as explicit row-major reductions
instead of calls to `F.avg_pool2d` / `F.max_pool2d`.  It states the arithmetic `tdx_coarse_epilogue` implements, and
tests/test_coarse_pooling_cpu.py pins it bit for bit to the reference's own code (tests/golden/coarse_pool_golden.npz):

  v = x / sigma_data * stds + means;  v[1] = v[0] - v[1];  pool by n;  out = cat([v w, w])

  avg  sum from +0 over the n x n cells in row-major order, divided once by n*n
  max  start at -inf, take a cell that is greater or NaN (NaN propagates; of equal values, +-0 included, the first stays)
  min  -max(-x)

Channel 0 pools by `elev_mode`, channel 1 by `p5_mode` ('max', 'min', anything else averages), channels 2-5 average.
n == 1 does not pool."""
from __future__ import annotations

import torch


def _reduce(cells: torch.Tensor, mode) -> torch.Tensor:
    """cells [h, w, n*n] in row-major window order -> [h, w]."""
    if mode == "min":
        return -_reduce(-cells, "max")
    if mode == "max":
        acc = torch.full(cells.shape[:-1], float("-inf"), dtype=torch.float32)
        for k in range(cells.shape[-1]):
            u = cells[..., k]
            acc = torch.where((u > acc) | torch.isnan(u), u, acc)
        return acc
    acc = torch.zeros(cells.shape[:-1], dtype=torch.float32)
    for k in range(cells.shape[-1]):
        acc = acc + cells[..., k]
    return acc / float(cells.shape[-1])


def pool(v: torch.Tensor, n: int, elev_mode="avg", p5_mode="avg") -> torch.Tensor:
    """[6, H, W] de-normalised coarse channels -> [6, H/n, W/n]."""
    if n == 1:
        return v
    c, h, w = v.shape
    cells = v.reshape(c, h // n, n, w // n, n).permute(0, 1, 3, 2, 4).reshape(c, h // n, w // n, n * n)
    modes = [elev_mode, p5_mode] + ["avg"] * (c - 2)
    return torch.stack([_reduce(cells[k], modes[k]) for k in range(c)])


def epilogue(x, means, stds, window, n: int, elev_mode="avg", p5_mode="avg", sigma_data: float = 0.5) -> torch.Tensor:
    """[6, 64, 64] raw solve output -> the packed [7, 64/n, 64/n] coarse tile."""
    x = torch.as_tensor(x, dtype=torch.float32)
    means = torch.as_tensor(means, dtype=torch.float32).view(-1, 1, 1)
    stds = torch.as_tensor(stds, dtype=torch.float32).view(-1, 1, 1)
    window = torch.as_tensor(window, dtype=torch.float32)
    v = x / sigma_data * stds + means
    v[1] = v[0] - v[1]
    v = pool(v, n, elev_mode, p5_mode)
    return torch.cat([v * window[None], window[None]])
