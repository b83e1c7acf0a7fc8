"""Unbounded, lazy, device-resident canvas -- the arithmetic and window protocol of the reference's external canvas
engine (`infinite_tensor>=0.3.0`, requirements.txt:32; absent from the reference checkout), as observable from its call sites
(world_pipeline.py:982-992,1146-1201,1259-1270; annotated_infinite_panorama.py:141-226; SURVEY.md Appendix C):

  * `TensorWindow(size, stride, offset)`: window index k along an axis covers [k*stride+offset, k*stride+offset+size);
  * slicing `canvas[:, a:b, c:d]` (integers are real, possibly negative, world coordinates) returns the SUM over all
    windows intersecting the slice of f's outputs, computing missing windows on demand; each window's f receives the
    slices of its dependencies taken at the SAME window index through their own TensorWindow;
  * with `batch_size`, f receives lists of up to that many window indices (and lists of dependency slices).

PARITY UNPINNED against the library itself (it is not on disk and the reference has no tests for it); the semantics
above are pinned by tests/test_lazy_canvas_gpu.py against a brute-force evaluation, and the arithmetic (fp32 sums in
row-major window order) by the bounded-canvas tests.  Everything stays in HBM: every computed window is an fp32 CUDA tile
(byte-limited LRU, recompute on miss), a slice is assembled by adding its windows with tdx_canvas_add.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass

import torch

from .. import _lib as L
from .tiling import window_range


@dataclass(frozen=True)
class TensorWindow:
    size: tuple      # (C, h, w)
    stride: tuple    # (C, sh, sw)
    offset: tuple = (0, 0, 0)


class LazyCanvas:
    """cache_limit (bytes, None = unbounded): the computed windows are kept as fp32 tiles in HBM, least recently used
    first out, like the reference's `MemoryTileStore(cache_size_bytes)` (world_pipeline.py:666-674); a window that was
    evicted is simply recomputed by `f` the next time a slice needs it (f is deterministic: tile-seeded noise).  The
    cache is trimmed after a request has been served, so a limit smaller than one request's windows only means that
    the oldest of them are not kept."""

    def __init__(self, channels: int, f, output_window: TensorWindow, device, args=(), args_windows=(),
                 batch_size: int | None = None, block: int = 512, cache_limit: int | None = None):
        self.channels = channels
        self.f = f
        self.win = output_window
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise L.TdxError("LazyCanvas lives in GPU memory; there is no CPU path")
        self.args, self.args_windows = tuple(args), tuple(args_windows)
        assert len(self.args) == len(self.args_windows)
        self.batch_size = batch_size
        self.block = block                      # kept for API compatibility (storage is per window now)
        self.cache_limit = None if cache_limit is None else int(cache_limit)
        self.tiles: OrderedDict = OrderedDict()  # (i, j) -> fp32 [C, h, w] window output, in LRU order
        self.cache_bytes = 0
        self.windows_computed = 0
        self.windows_evicted = 0

    # ------------------------------------------------------------------ storage
    @property
    def done(self):
        """Window indices currently cached."""
        return self.tiles.keys()

    def _store(self, ij, tile: torch.Tensor):
        tile = tile.to(self.device, torch.float32).contiguous()
        assert tuple(tile.shape) == tuple(self.win.size), (tuple(tile.shape), self.win.size)
        self.tiles[ij] = tile
        self.cache_bytes += tile.numel() * 4
        self.windows_computed += 1

    def _evict(self, protect=()):
        if self.cache_limit is None:
            return
        protect = set(protect)
        for ij in list(self.tiles.keys()):
            if self.cache_bytes <= self.cache_limit:
                break
            if ij in protect:
                continue
            t = self.tiles.pop(ij)
            self.cache_bytes -= t.numel() * 4
            self.windows_evicted += 1

    def clear_cache(self):
        self.tiles.clear()
        self.cache_bytes = 0

    # ------------------------------------------------------------------ windows
    def window_origin(self, i: int, j: int) -> tuple[int, int]:
        return (i * self.win.stride[1] + self.win.offset[1], j * self.win.stride[2] + self.win.offset[2])

    def windows_for(self, a: int, b: int, c: int, d: int) -> list[tuple[int, int]]:
        """Window indices (row-major) whose extent intersects rows [a,b) x columns [c,d)."""
        rows = window_range(a, b, self.win.size[1], self.win.stride[1], self.win.offset[1])
        cols = window_range(c, d, self.win.size[2], self.win.stride[2], self.win.offset[2])
        return [(i, j) for i in rows for j in cols]

    def _dep_slices(self, i, j):
        out = []
        for dep, w in zip(self.args, self.args_windows):
            y0 = i * w.stride[1] + w.offset[1]
            x0 = j * w.stride[2] + w.offset[2]
            out.append(dep[:, y0:y0 + w.size[1], x0:x0 + w.size[2]])
        return out

    def _prefetch_deps(self, missing):
        """Before the windows `missing` are evaluated one (batch) at a time, make every dependency canvas compute ALL
        the windows they will read in one request: the union, row-major, so a dependency with `batch_size` fills its
        batches (a 512^2 read used to reach the latent stage as ~50 calls of 2-3 windows instead of ~8 of 16).  Exactly
        the windows the per-window reads would compute -- no more; skipped when the union would not fit the
        dependency's cache limit (the reads then compute on demand as before)."""
        for dep, w in zip(self.args, self.args_windows):
            if not isinstance(dep, LazyCanvas):
                continue
            need = set()
            for (i, j) in missing:
                y0 = i * w.stride[1] + w.offset[1]
                x0 = j * w.stride[2] + w.offset[2]
                need.update(dep.windows_for(y0, y0 + w.size[1], x0, x0 + w.size[2]))
            need = sorted(need)
            tile_bytes = 4 * dep.win.size[0] * dep.win.size[1] * dep.win.size[2]
            if dep.cache_limit is not None and len(need) * tile_bytes > dep.cache_limit:
                continue
            dep._ensure(need)

    def _ensure(self, idxs):
        missing = [ij for ij in idxs if ij not in self.tiles]
        if not missing:
            return
        if len(missing) > 1 and self.args:
            self._prefetch_deps(missing)
        if self.batch_size is None:
            for (i, j) in missing:
                self._store((i, j), self.f((0, i, j), *self._dep_slices(i, j)))
        else:
            for g0 in range(0, len(missing), self.batch_size):
                grp = missing[g0:g0 + self.batch_size]
                deps = [self._dep_slices(i, j) for (i, j) in grp]
                lists = [list(col) for col in zip(*deps)] if deps and deps[0] else []
                tiles = self.f([(0, i, j) for (i, j) in grp], *lists)
                for ij, tile in zip(grp, tiles):
                    self._store(ij, tile)

    # ------------------------------------------------------------------ read
    def __getitem__(self, key) -> torch.Tensor:
        if not (isinstance(key, tuple) and len(key) == 3):
            raise IndexError("LazyCanvas is indexed as canvas[:, a:b, c:d]")
        cs, ys, xs = key
        a, b, c, d = ys.start, ys.stop, xs.start, xs.stop
        if None in (a, b, c, d) or b <= a or d <= c:
            raise IndexError("row and column slices need explicit start < stop (world coordinates, may be negative)")
        idxs = self.windows_for(a, b, c, d)
        self._ensure(idxs)
        # the slice = sum of the covering windows in row-major window order (the order of the bounded samplers and of
        # oracle/tiling.py), whatever the order they were computed in: reads are reproducible bit for bit
        out = torch.zeros((self.channels, b - a, d - c), dtype=torch.float32, device=self.device)
        _, th, tw = self.win.size
        for (i, j) in idxs:
            tile = self.tiles[(i, j)]
            self.tiles.move_to_end((i, j))
            y0, x0 = self.window_origin(i, j)
            L.call(L.lib().tdx_canvas_add, self.device, out.data_ptr(), self.channels, b - a, d - c, tile.data_ptr(),
                   th, tw, y0 - a, x0 - c)
        self._evict()          # trim to the limit: the windows just used are the most recent, the oldest go first
        return out[cs]
