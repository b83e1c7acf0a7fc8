"""The explorer's detail view on the device (terrain_diffusion/inference/explorer/server.py:188-270).

`GET /api/detail.png` renders a window as an elevation image (`terrain` colormap), a temperature image (`RdBu_r`) or
the shaded relief, and `GET /api/detail_raw` sends the window as int16 elevation + fp32 temperature.  The reference
copies get()'s elevation and all five climate planes to the host for either, then runs np.nanmin / np.nanmax,
matplotlib's Normalize and colormap and `to_rgba(bytes=True)` there.  Here csrc/tdx_explorer.cu does that work after
get()'s device read-out, and the caller copies one uint8 image or one body to the host.  PNG encoding stays on the host.

The colormap tables are matplotlib's, restated without matplotlib: `terrain` is `relief.terrain_lut`, and `RdBu_r`
is built the way matplotlib builds it -- `LinearSegmentedColormap.from_list` of the 11 ColorBrewer RdBu colours, then
`reversed()`, which rebuilds the table from the mirrored segments (1 - x, y1, y0).
"""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib as L
from . import postproc
from .relief import LUT_SIZE, create_lookup_table, terrain_lut

# matplotlib/_cm.py `_RdBu_data`: ColorBrewer RdBu, 11 classes, as 8-bit RGB
RDBU_HEX = ("67001f", "b2182b", "d6604d", "f4a582", "fddbc7", "f7f7f7", "d1e5f0", "92c5de", "4393c3", "2166ac",
            "053061")


def rdbu_r_lut() -> np.ndarray:
    """fp64 [256, 3]: `plt.get_cmap('RdBu_r')`'s table.  RdBu is `from_list` of RDBU_HEX (k / 255) at
    linspace(0, 1, 11); `reversed()` lists each channel's segments (1 - x, y1, y0) in reverse order and runs
    `_create_lookup_table` again.  1 - x is not always the mirrored position of linspace, so this is not RdBu's finished
    table flipped."""
    rgb = np.array([[int(h[k:k + 2], 16) / 255 for k in (0, 2, 4)] for h in RDBU_HEX], dtype=np.float64)
    vals = np.linspace(0, 1, len(RDBU_HEX))
    out = np.empty((LUT_SIZE, 3), dtype=np.float64)
    for c in range(3):
        seg = np.column_stack([vals, rgb[:, c], rgb[:, c]])
        out[:, c] = create_lookup_table([(1.0 - x, y1, y0) for x, y0, y1 in reversed(seg)])
    return out


CMAPS = {"terrain": terrain_lut, "RdBu_r": rdbu_r_lut}
_luts: dict = {}


def _lut_on(cmap: str, device: torch.device) -> torch.Tensor:
    """The colormap's table rounded to fp32 (the reference's `.astype(np.float32)` of the RGBA), cached per device."""
    if (cmap, device) not in _luts:
        _luts[(cmap, device)] = torch.from_numpy(CMAPS[cmap]().astype(np.float32)).to(device)
    return _luts[(cmap, device)]


def detail_window(i1, j1, i2, j2, mode: str = "elevation") -> tuple[int, int]:
    """(H, W) of a detail request after the terrain API's checks at scale 1 (`postproc.terrain_window`: ints, a
    non-empty window, at most 65535 rows; ValueError).  The relief needs H, W >= 2 (np.gradient)."""
    postproc.terrain_window(i1, j1, i2, j2, 1)
    H, W = int(i2) - int(i1), int(j2) - int(j1)
    if mode not in ("elevation", "temperature") and (H < 2 or W < 2):
        raise ValueError(f"the relief needs a window of at least 2 x 2 pixels (np.gradient), got {H} x {W}")
    return H, W


def colour_image(plane: torch.Tensor, cmap: str) -> torch.Tensor:
    """Two launches on the plane's device: the NaN-ignoring range into a device buffer, then the colour pass that reads
    it.  CUDA fp32 [H, W] -> CUDA uint8 [H, W, 4]."""
    plane = postproc.check_plane(plane, "colour_plane")
    dev = plane.device
    rng = torch.empty(2, dtype=torch.int32, device=dev)
    out = torch.empty((*plane.shape, 4), dtype=torch.uint8, device=dev)
    n = plane.numel()
    L.call(L.lib().tdx_detail_range, dev, plane.data_ptr(), n, rng.data_ptr())
    L.call(L.lib().tdx_detail_colour, dev, plane.data_ptr(), n, rng.data_ptr(), _lut_on(cmap, dev).data_ptr(),
           out.data_ptr())
    return out


def colour_plane(plane, cmap: str):
    """The elevation / temperature image of `/api/detail.png` (server.py:206-218 and `_png_response`) for any fp32
    plane: vmin, vmax = nanmin, nanmax (vmax = vmin + 1 when equal), matplotlib's Normalize and the colormap `cmap`
    ('terrain' or 'RdBu_r'), then the uint8 RGBA that `plt.imsave` hands to the PNG encoder.  NaN pixels are
    (0, 0, 0, 0); an all-NaN plane is all (0, 0, 0, 0); where vmin + 1 == vmin (|vmin| >= 2^53) every pixel, NaN
    included, takes the first colour, as Normalize fills 0.

    A CUDA tensor gives a CUDA uint8 [H, W, 4] tensor on its device; a numpy array or CPU tensor is computed on the
    current CUDA device and gives a numpy array.  Raises ValueError for an unknown colormap or a plane that is not
    two-dimensional and non-empty."""
    if cmap not in CMAPS:
        raise ValueError(f"colour_plane: colormap {cmap!r} is not restated; use one of {sorted(CMAPS)}")
    shape = tuple(plane.shape) if hasattr(plane, "shape") else np.shape(plane)
    if len(shape) != 2 or 0 in shape:
        raise ValueError(f"colour_plane: expected a non-empty [H, W] plane, got shape {shape}")
    if isinstance(plane, torch.Tensor) and plane.is_cuda:
        return colour_image(plane.detach().float(), cmap)
    if not torch.cuda.is_available():
        raise L.TdxError("colour_plane runs on a CUDA device and none is available (there is no CPU path)")
    host = plane.detach().cpu().numpy() if isinstance(plane, torch.Tensor) else np.asarray(plane)
    return colour_image(torch.from_numpy(np.ascontiguousarray(host, dtype=np.float32)).cuda(), cmap).cpu().numpy()


def relief_rgba8(rgb: torch.Tensor) -> torch.Tensor:
    """The relief image of `/api/detail.png` (server.py:223-228 and `_png_response`): CUDA fp32 RGB [H, W, 3] ->
    CUDA uint8 RGBA [H, W, 4], alpha 255; a pixel with a NaN channel is (0, 0, 0, 0)."""
    if not (isinstance(rgb, torch.Tensor) and rgb.is_cuda and rgb.dtype == torch.float32 and rgb.dim() == 3
            and rgb.shape[2] == 3 and rgb.numel() > 0):
        raise L.TdxError(f"relief_rgba8: expected a non-empty CUDA float32 [H, W, 3] tensor, got "
                         f"{getattr(rgb, 'device', None)} {getattr(rgb, 'dtype', None)} {tuple(getattr(rgb, 'shape', ()))}")
    rgb = rgb.contiguous()
    out = torch.empty((rgb.shape[0], rgb.shape[1], 4), dtype=torch.uint8, device=rgb.device)
    L.call(L.lib().tdx_detail_rgba8, rgb.device, rgb.data_ptr(), rgb.shape[0] * rgb.shape[1], out.data_ptr())
    return out


def raw_body(elev: torch.Tensor, temp: torch.Tensor | None) -> torch.Tensor:
    """The `/api/detail_raw` body (server.py:252-260) in one launch: CUDA uint8 [2HW (+ 4HW)] = H*W int16-LE elevations
    (floor, clip, NaN -> 0, as `terrain_payload` packs them), then temp's H*W fp32-LE values bit for bit."""
    elev = postproc.check_plane(elev, "raw_body(elev)")
    if temp is not None:
        temp = postproc.check_plane(temp, "raw_body(temp)", tuple(elev.shape), elev.device)
    n = elev.numel()
    body = torch.empty((n * (6 if temp is not None else 2),), dtype=torch.uint8, device=elev.device)
    L.call(L.lib().tdx_detail_raw, elev.device, elev.data_ptr(), None if temp is None else temp.data_ptr(), n,
           body.data_ptr())
    return body
