"""EDMUnet2D -- drop-in for terrain_diffusion.models.edm_unet.EDMUnet2D (reference edm_unet.py:15-193) whose forward
runs on hand-written sm_90a kernels through libtdx (see plan.py for how blocks map to launches).

Same constructor arguments, same parameter names/shapes (reference checkpoints load with load_state_dict /
from_pretrained), same call signature `model(x, noise_labels, conditional_inputs, return_logvar=False,
precomputed_embeds=None)`, `.config`, `.eval()`, `.to()`, `.parameters()`.  Inference only: there is no autograd
through the CUDA path and NO CPU / PyTorch fallback -- a CPU tensor or a missing libtdx.so raises.
"""
from __future__ import annotations

import json
import math
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn

from .. import _lib as L
from .plan import FoldedWeights, UNetEmitter, UNetProgram, block_plan


class _AttrDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e


class _Weight(nn.Module):
    """Parameter holder named like the reference's MPConv / MPEmbedding (`.weight`)."""

    def __init__(self, *shape):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(*shape))


class _Fourier(nn.Module):
    def __init__(self, num_channels, s=1, positional=False):
        super().__init__()
        if positional:
            half = num_channels // 2
            self.register_buffer("freqs", torch.exp(torch.arange(half) * -(math.log(10) / (half - 1))))
        else:
            self.register_buffer("freqs", 2 * np.pi * torch.randn(num_channels) * s)
            self.register_buffer("phases", 2 * np.pi * torch.rand(num_channels))
        self.positional = positional

    def forward(self, x):
        y = x.to(torch.float32).outer(self.freqs.to(torch.float32))
        if self.positional:
            return (torch.cat([torch.sin(y), torch.cos(y)], dim=1) * np.sqrt(2)).to(x.dtype)
        return ((y + self.phases.to(torch.float32)).cos() * np.sqrt(2)).to(x.dtype)


class _Block(nn.Module):
    def __init__(self, cin, cout, emb_channels, mode, attention_heads):
        super().__init__()
        self.emb_gain = nn.Parameter(torch.zeros([]))
        self.conv_res0 = _Weight(cout, cout if mode == "enc" else cin, 3, 3)
        if emb_channels > 0:
            self.emb_linear = _Weight(cout, emb_channels)
        self.conv_res1 = _Weight(cout, cout, 3, 3)
        if cin != cout:
            self.conv_skip = _Weight(cout, cin, 1, 1)
        if attention_heads:
            self.attn_qkv = _Weight(cout * 3, cout, 1, 1)
            self.attn_proj = _Weight(cout, cout, 1, 1)


def _host_mp_silu(x):
    return torch.nn.functional.silu(x) / 0.596


class EDMUnet2D(nn.Module):
    config_name = "config.json"

    def __init__(self, image_size, in_channels, out_channels=None, model_channels=128, model_channel_mults=None,
                 layers_per_block=2, emb_channels=None, noise_emb_dims=None, attn_resolutions=None,
                 midblock_attention=True, concat_balance=0.3, logvar_channels=128, block_kwargs=None,
                 conditional_inputs=[], encode_only=False, disable_out_gain=False, fourier_scale=1, n_logvar=1):
        super().__init__()
        self._internal_dict = _AttrDict(
            image_size=image_size, in_channels=in_channels, out_channels=out_channels, model_channels=model_channels,
            model_channel_mults=model_channel_mults, layers_per_block=layers_per_block, emb_channels=emb_channels,
            noise_emb_dims=noise_emb_dims, attn_resolutions=attn_resolutions, midblock_attention=midblock_attention,
            concat_balance=concat_balance, logvar_channels=logvar_channels, block_kwargs=block_kwargs,
            conditional_inputs=conditional_inputs, encode_only=encode_only, disable_out_gain=disable_out_gain,
            fourier_scale=fourier_scale, n_logvar=n_logvar)
        cfg = self._internal_dict
        if encode_only:
            raise NotImplementedError("encode_only models are not part of the sampling hot path")
        self.concat_balance = concat_balance
        mults = model_channel_mults or [1, 2, 3, 4]
        emb_ch = emb_channels or model_channels * max(mults)
        noise_dims = model_channels if noise_emb_dims is None else noise_emb_dims
        self.emb_channels = emb_ch
        if noise_dims == 0 and len(conditional_inputs) == 0:
            emb_ch = 0
            self.emb_channels = 0
        positional = fourier_scale == "pos"
        if noise_dims > 0:
            self.noise_fourier = _Fourier(noise_dims, s=1 if positional else fourier_scale, positional=positional)
            self.noise_linear = _Weight(emb_ch, noise_dims)
        else:
            self.noise_fourier = None
            self.noise_linear = None
        self.conditional_layers = nn.ModuleList([])
        self.conditional_weights = [1] if self.noise_linear is not None else []
        self._cond_kinds = []
        for kind, x, weight in conditional_inputs:
            if kind == "float":
                self.conditional_layers.append(nn.Sequential(_Fourier(x), _Weight(emb_ch, x)))
            elif kind == "tensor":
                self.conditional_layers.append(_Weight(emb_ch, x))
            elif kind == "embedding":
                self.conditional_layers.append(_Weight(x, emb_ch))
            else:
                raise ValueError(f"unknown conditional input type {kind!r}")
            self._cond_kinds.append(kind)
            self.conditional_weights.append(weight)
        if not disable_out_gain:
            self.out_gain = nn.Parameter(torch.zeros([]))
        else:
            self.out_gain = 1.0
        enc, dec = block_plan(cfg)
        cph = (block_kwargs or {}).get("channels_per_head", 64)
        self.enc = nn.ModuleDict()
        for b in enc:
            if b["kind"] == "conv":
                self.enc[b["name"]] = _Weight(b["cout"], b["cin"], 3, 3)
            else:
                self.enc[b["name"]] = _Block(b["cin"], b["cout"], emb_ch, "enc",
                                             b["cout"] // cph if b["attention"] else 0)
        self.dec = nn.ModuleDict()
        for b in dec:
            self.dec[b["name"]] = _Block(b["cin"], b["cout"], emb_ch, "dec", b["cout"] // cph if b["attention"] else 0)
        self.out_conv = _Weight(out_channels or in_channels, (dec[-1] if dec else enc[-1])["cout"], 3, 3)
        self.logvar_fourier = _Fourier(logvar_channels)
        self.logvar_linear = _Weight(n_logvar, logvar_channels)
        self._folded = None
        self._plans: dict = {}
        self.max_cached_plans = 8
        self.use_cuda_graph = True

    # ------------------------------------------------------------------ diffusers-like surface
    @property
    def config(self):
        return self._internal_dict

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def count_parameters(self):
        return sum(p.numel() for p in self.parameters())

    def _apply(self, fn, *a, **k):
        self.invalidate()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self.invalidate()
        return super().load_state_dict(*a, **k)

    def invalidate(self):
        """Drop folded weights and compiled programs (call after changing parameters)."""
        self._folded = None
        self._plans = {}

    @classmethod
    def from_config(cls, config: dict):
        cfg = {k: v for k, v in dict(config).items() if not k.startswith("_")}
        return cls(**cfg)

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **_unused):
        """diffusers layout: <path>/<subfolder>/config.json + diffusion_pytorch_model.safetensors (or .bin)."""
        root = Path(path) / subfolder if subfolder else Path(path)
        if not (root / cls.config_name).exists():
            raise FileNotFoundError(f"{root / cls.config_name} not found (offline: local directories only)")
        model = cls.from_config(json.loads((root / cls.config_name).read_text()))
        st = root / "diffusion_pytorch_model.safetensors"
        if st.exists():
            from safetensors.torch import load_file
            sd = load_file(str(st))
        else:
            sd = torch.load(root / "diffusion_pytorch_model.bin", map_location="cpu")
        model.load_state_dict(sd)
        return model.eval()

    def save_pretrained(self, path):
        from safetensors.torch import save_file
        root = Path(path)
        root.mkdir(parents=True, exist_ok=True)
        (root / self.config_name).write_text(json.dumps(dict(self.config), indent=2))
        save_file({k: v.contiguous() for k, v in self.state_dict().items()},
                  str(root / "diffusion_pytorch_model.safetensors"))

    # ------------------------------------------------------------------ embeddings (conditional models: host side)
    def _host_embedding(self, noise_labels, conditional_inputs):
        """compute_embeddings (edm_unet.py:145-159) for conditional models: a handful of fp32 GEMVs on the model's
        device with the weights folded once (FoldedWeights); rows = noise_labels.numel() (all the steps of a solve in
        one call)."""
        g = self.folded().g
        embeds = []
        if self.noise_linear is not None:
            embeds.append(self.noise_fourier(noise_labels.float()) @ g["noise_linear"])
        for i, (layer, kind, inp) in enumerate(zip(self.conditional_layers, self._cond_kinds, conditional_inputs)):
            if kind == "float":
                embeds.append(layer[0](inp.float()) @ g[f"cond{i}"])
            elif kind == "tensor":
                embeds.append(_host_mp_silu(inp.float() @ g[f"cond{i}"]))
            else:
                embeds.append(torch.nn.functional.embedding(inp, g[f"cond{i}"]))
        w = self.conditional_weights
        w32 = torch.tensor([float(v) for v in w], dtype=torch.float32)            # host: mp_sum's weights and their norm
        emb = sum(e * float(wi) for e, wi in zip(embeds, w32)) / float(torch.linalg.vector_norm(w32))
        return _host_mp_silu(emb)

    # ------------------------------------------------------------------ forward
    def folded(self) -> FoldedWeights:
        if self._folded is None:
            dev = self.device
            if dev.type != "cuda":
                raise L.TdxError("EDMUnet2D (GPU path) needs its parameters on a CUDA device; there is no CPU path")
            L.lib()
            self._folded = FoldedWeights(self, dev)
        return self._folded

    def _forward_plan(self, n, h, w, with_emb):
        key = ("fwd", n, h, w, with_emb)
        if key not in self._plans:
            fw = self.folded()
            dev = fw.device
            em = UNetEmitter(fw, n, h, w)
            bufs = SimpleNamespace(
                x=torch.zeros((n, fw.in_channels, h, w), dtype=torch.float32, device=dev),
                labels=torch.zeros((n,), dtype=torch.float32, device=dev),
                emb=torch.zeros((n, fw.emb_channels), dtype=torch.float32, device=dev) if with_emb else None,
                out=torch.zeros((n, fw.out_channels, h, w), dtype=torch.float32, device=dev))
            prog = UNetProgram(dev)
            em.emit_embed(prog, labels=bufs.labels, emb_in=bufs.emb)
            em.emit(prog, [(bufs.x, fw.in_channels, None)], model_out=bufs.out)
            self._plans[key] = (prog, bufs)
            while len(self._plans) > self.max_cached_plans:       # every plan owns a full activation arena + a graph
                self._plans.pop(next(iter(self._plans)))
        else:
            self._plans[key] = self._plans.pop(key)               # most recently used last
        return self._plans[key]

    @torch.no_grad()
    def forward(self, x, noise_labels, conditional_inputs=None, return_logvar=False, precomputed_embeds=None):
        conditional_inputs = conditional_inputs or []
        assert len(conditional_inputs) == len(self.conditional_layers), "Invalid number of conditional inputs"
        if self.training:
            raise L.TdxError("the GPU path is inference-only: call model.eval()")
        if x.device.type != "cuda":
            raise L.TdxError("EDMUnet2D (GPU path) got a CPU tensor; there is no CPU fallback")
        n, c, h, w = x.shape
        needs_host_emb = precomputed_embeds is not None or len(self.conditional_layers) > 0 or \
            not (self.noise_fourier is not None and self.noise_fourier.positional)
        prog, bufs = self._forward_plan(n, h, w, needs_host_emb)
        bufs.x.copy_(x)
        if needs_host_emb:
            emb = precomputed_embeds if precomputed_embeds is not None else \
                self._host_embedding(noise_labels, conditional_inputs)
            bufs.emb.copy_(emb)
        else:
            bufs.labels.copy_(noise_labels.reshape(-1).expand(n) if noise_labels.numel() == 1 else noise_labels)
        prog.run(self.use_cuda_graph)
        out = bufs.out.to(x.dtype, copy=True)
        if return_logvar:
            from .plan import effective_weight
            lv = self.logvar_fourier(torch.log(torch.tan(noise_labels.float()) / 8)) @ \
                effective_weight(self.logvar_linear.weight).T
            return out, lv.reshape(-1, 1, 1, 1).to(x.dtype)
        return out

    def norm_weights(self):
        """Reference training hook (edm_unet.py:189-192); weights are re-normalised at fold time here."""
        return None
