"""Record the launch descriptors the product's U-Net programs are made of, without a GPU and without an activation arena.

The weights are folded onto the meta device and every buffer the emitter owns is a stand-in with a distinct, non-zero
address, so a recorded descriptor still tells which side planes (rms_out, resid_inv) a launch uses, and which buffer
it writes (`RecordingProgram.key_of`).
"""
from __future__ import annotations

import torch

from oracle import unet as ounet
from terrain_diffusion_b200.models import EDMUnet2D
from terrain_diffusion_b200.models.plan import FoldedWeights, UNetEmitter, UNetProgram

BASE_CFG = dict(image_size=512, in_channels=5, out_channels=5, model_channels=192, model_channel_mults=[1, 2, 3, 4],
                layers_per_block=3, attn_resolutions=[8, 16], midblock_attention=True, concat_balance=0.5,
                conditional_inputs=[["tensor", 58, 1.0]], fourier_scale="pos", block_kwargs={"dropout": 0.1})
"""The latent (base) model, 192 x [1, 2, 3, 4] with self-attention at 8^2 / 16^2."""
GUIDE_CFG = dict(BASE_CFG, model_channels=128)
"""The 128-channel guide of the two-model guided base diffusion."""
COARSE_CFG = dict(image_size=16, in_channels=11, out_channels=6, model_channels=128, model_channel_mults=[1],
                  layers_per_block=2, attn_resolutions=[], midblock_attention=False, concat_balance=0.5,
                  conditional_inputs=[["float", 64, 0.2]] * 5, fourier_scale="pos", block_kwargs={})
CONFIGS = {"decoder": ounet.DECODER_CFG, "base": BASE_CFG, "guide": GUIDE_CFG, "coarse": COARSE_CFG}


class _StandIn:
    """Takes the place of a device buffer: only its address is ever read while emitting."""

    def __init__(self, addr):
        self.addr = addr

    def data_ptr(self):
        return self.addr


class RecordingProgram(UNetProgram):
    """A UNetProgram that keeps a copy of every launch descriptor instead of handing it to the library."""

    def __init__(self):
        self.handle = None
        self.keep: list = []
        self.arena: dict = {}
        self.n_igemm = 0
        self.n_launch = 0
        self.launches: list = []       # [(kind, descriptor copy)]
        self.key_of: dict = {}         # stand-in address -> emitter buffer key

    def add(self, kind, desc):
        self.launches.append((kind, type(desc).from_buffer_copy(desc)))
        self.keep.append(desc)         # keeps what the descriptor points to (the embed block array) alive
        self.n_launch += 1
        if kind == "igemm":
            self.n_igemm += 1

    def igemm(self):
        return [d for k, d in self.launches if k == "igemm"]


class RecordingEmitter(UNetEmitter):
    def __init__(self, fw, n, h, w, prog: RecordingProgram):
        super().__init__(fw, n, h, w)
        self._prog = prog
        self._next = 1 << 40

    def _buffer(self, shape, dtype, fill=None):
        nbytes = torch.empty((), dtype=dtype).element_size()
        for s in shape:
            nbytes *= s
        buf = _StandIn(self._next)
        self._next += (nbytes + 255) // 256 * 256
        return buf

    def act(self, key, c, h, w):
        new = key not in self.arena
        t = super().act(key, c, h, w)
        if new:
            self._prog.key_of[t.data_ptr()] = key
        return t


_FOLDED: dict = {}


def folded(name: str) -> FoldedWeights:
    """The model's weights folded onto the meta device (shapes only; cached per model)."""
    if name not in _FOLDED:
        torch.manual_seed(0)
        _FOLDED[name] = FoldedWeights(EDMUnet2D(**CONFIGS[name]).eval(), torch.device("meta"))
    return _FOLDED[name]


def capture_forward(name: str, n: int, hw: int) -> RecordingProgram:
    """Every launch of one forward of model `name` on n images of hw x hw, as EDMUnet2D.forward plans it."""
    fw = folded(name)
    prog = RecordingProgram()
    em = RecordingEmitter(fw, n, hw, hw, prog)
    meta = torch.device("meta")
    if fw.has_cond or not fw.pos_emb:
        em.emit_embed(prog, emb_in=torch.empty((n, fw.emb_channels), device=meta))
    else:
        em.emit_embed(prog, labels=torch.empty((n,), device=meta))
    x = torch.empty((n, fw.in_channels, hw, hw), device=meta)
    em.emit(prog, [(x, fw.in_channels, None)], model_out=torch.empty((n, fw.out_channels, hw, hw), device=meta))
    return prog


def layer_of(prog: RecordingProgram, d) -> str:
    """The emitter key of the buffer a recorded igemm launch writes first (names the layer)."""
    return prog.key_of.get(d.out[0].ptr, "?")
