"""Device-resident overlap-sum canvas: the arithmetic the reference delegates to the external `infinite_tensor`
package ("sums overlapping window outputs; dividing the first C channels by the last recovers the weighted average",
annotated_infinite_panorama.py:141-146) and restates on bounded canvases at
training/evaluation/sample_diffusion_decoder.py:122-125 and evaluation/infinite_consistency.py:236-239.

fp32 planes (sum of x*w per channel, sum of w) live in HBM; tiles are accumulated by a vectorisable fp32 kernel with
separately rounded multiply and add, so replaying tiles in the reference's row-major order is bit-identical to it.
"""
from __future__ import annotations

import torch

from .. import _lib as L
from .tiling import linear_weight_window


class BlendCanvas:
    def __init__(self, channels: int, height: int, width: int, device, origin=(0, 0)):
        if torch.device(device).type != "cuda":
            raise L.TdxError("BlendCanvas lives in GPU memory; there is no CPU path")
        self.channels, self.height, self.width = channels, height, width
        self.origin = origin  # canvas coordinate of element [0, 0] (supports negative world coordinates)
        self.val = torch.zeros((channels, height, width), dtype=torch.float32, device=device)
        self.wsum = torch.zeros((height, width), dtype=torch.float32, device=device)
        self._windows: dict = {}

    def window(self, size: int) -> torch.Tensor:
        if size not in self._windows:
            self._windows[size] = linear_weight_window(size, self.val.device).contiguous()
        return self._windows[size]

    def clear(self):
        self.val.zero_()
        self.wsum.zero_()

    def accumulate(self, tile: torch.Tensor, y0: int, x0: int, window: torch.Tensor | None = None):
        """tile: fp32 [C, th, tw] on the canvas device; (y0, x0): world coordinates of its top-left pixel.  window: fp32
        [th, tw] blend weights on the canvas device (any strides); None: the linear window, for square tiles only."""
        c, th, tw = tile.shape
        assert c == self.channels and tile.dtype == torch.float32 and tile.is_cuda
        tile = tile.contiguous()
        if window is None:
            if th != tw:
                raise ValueError(f"a {th}x{tw} tile needs an explicit [{th}, {tw}] window (the default is square)")
            win = self.window(th)
        else:
            if tuple(window.shape) != (th, tw) or window.dtype != torch.float32 or window.device != self.val.device:
                raise ValueError(f"window must be fp32 [{th}, {tw}] on {self.val.device}; got {window.dtype} "
                                 f"{list(window.shape)} on {window.device}")
            win = window.contiguous()
        L.call(L.lib().tdx_blend_accumulate, self.val.device, self.val.data_ptr(), self.wsum.data_ptr(), c, self.height,
               self.width, tile.data_ptr(), win.data_ptr(), th, tw, y0 - self.origin[0], x0 - self.origin[1])

    def packed(self) -> torch.Tensor:
        """[C+1, H, W] un-normalised (sum x*w, sum w) -- what slicing a reference InfiniteTensor returns."""
        return torch.cat([self.val, self.wsum[None]], dim=0)

    def normalized(self, divisor: float = 1.0) -> torch.Tensor:
        out = torch.empty_like(self.val)
        L.call(L.lib().tdx_blend_normalize, self.val.device, out.data_ptr(), self.val.data_ptr(), self.wsum.data_ptr(),
               self.channels, self.height * self.width, float(divisor))
        return out
