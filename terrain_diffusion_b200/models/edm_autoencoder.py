"""EDMAutoencoder -- drop-in for terrain_diffusion.models.edm_autoencoder.EDMAutoencoder (reference
edm_autoencoder.py:13-167), the model that defines the latent space: `preencode` and `decode` run on hand-written
sm_90a kernels through libtdx.

Same constructor arguments and parameter names / shapes (`encoder.*`, `decoder.{i}.*`, `decoder_conv.weight`,
`out_conv.weight`, `out_gain`, `logvar`), so reference checkpoints load with load_state_dict / from_pretrained.

  preencode   the encoder is an EDMUnet2D(encode_only=True): its own planned program (im2col first convolution, the
              encoder blocks, conv_out with the 2 x latent_channels means / logvars), replayed as one CUDA graph
  decode      one planned program too (plan.autoencoder_decoder_plan): the 1x1 decoder_conv over [z, ones] runs as the
              tensor-core first convolution with weights only on the centre tap, then the decoder-mode block chain
              (a 1x1 conv_skip becomes a K-slab of conv_res1), then out_conv with out_gain folded
  postencode  plain torch ops on the tensors' device, as the reference

Inference only, CUDA only, like EDMUnet2D: a CPU tensor or training mode raises.  `direct_skips` is not implemented on
the GPU path: preencode / decode of such a model raise NotImplementedError.
"""
from __future__ import annotations

import json
from pathlib import Path
from types import SimpleNamespace

import torch
import torch.nn as nn

from .. import _lib as L
from .edm_unet import EDMUnet2D, _AttrDict, _Block, _Weight
from .plan import FoldedWeights, UNetEmitter, UNetProgram, autoencoder_decoder_plan


class EDMAutoencoder(nn.Module):
    config_name = "config.json"

    def __init__(self, image_size, in_channels, out_channels=None, model_channels=128, model_channel_mults=None,
                 layers_per_block=3, layers_per_block_decoder=None, attn_resolutions=None, midblock_attention=True,
                 logvar_channels=128, block_kwargs=None, conditional_inputs=[], latent_channels=None, n_logvar=1,
                 direct_skips=[]):
        super().__init__()
        self._internal_dict = _AttrDict(
            image_size=image_size, in_channels=in_channels, out_channels=out_channels, model_channels=model_channels,
            model_channel_mults=model_channel_mults, layers_per_block=layers_per_block,
            layers_per_block_decoder=layers_per_block_decoder, attn_resolutions=attn_resolutions,
            midblock_attention=midblock_attention, logvar_channels=logvar_channels, block_kwargs=block_kwargs,
            conditional_inputs=conditional_inputs, latent_channels=latent_channels, n_logvar=n_logvar,
            direct_skips=direct_skips)
        assert latent_channels is not None, "latent_channels must be specified"
        mults = model_channel_mults or [1, 2, 3, 4]
        self.encoder = EDMUnet2D(
            image_size=image_size, in_channels=in_channels, out_channels=latent_channels * 2,
            model_channels=model_channels, model_channel_mults=mults, layers_per_block=layers_per_block,
            emb_channels=0, noise_emb_dims=0, attn_resolutions=attn_resolutions, midblock_attention=midblock_attention,
            logvar_channels=logvar_channels, block_kwargs=block_kwargs, conditional_inputs=conditional_inputs,
            encode_only=True, disable_out_gain=False)
        self.encoder.out_gain = nn.Parameter(torch.ones([]))
        self.decoder_conv = _Weight(model_channels * mults[-1], latent_channels + len(direct_skips) + 1, 1, 1)
        enc, dec = autoencoder_decoder_plan(self._decoder_config())
        cph = (block_kwargs or {}).get("channels_per_head", 64)
        self.decoder = nn.ModuleList(_Block(b["cin"], b["cout"], 0, "dec", b["cout"] // cph if b["attention"] else 0)
                                     for b in dec)
        self.out_conv = _Weight(out_channels or in_channels, dec[-1]["cout"], 3, 3)
        self.out_gain = nn.Parameter(torch.ones([]) * 0.1)
        self.logvar = nn.Parameter(torch.zeros([n_logvar]))
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
        return sum(p.numel() for p in self.parameters() if p.requires_grad)

    def _apply(self, fn, *a, **k):
        self.invalidate()
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self.invalidate()
        return super().load_state_dict(*a, **k)

    def invalidate(self):
        """Drop folded weights and compiled programs of the encoder and the decoder (call after changing parameters)."""
        self.encoder.invalidate()
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

    # ------------------------------------------------------------------ GPU path
    def _decoder_config(self) -> dict:
        """The decoder as an EDMUnet2D-like config for the planner: latents in, no embedding, no skip concatenation."""
        c = self.config
        return dict(c, in_channels=c["latent_channels"], out_channels=c["out_channels"] or c["in_channels"],
                    noise_emb_dims=0, emb_channels=0, conditional_inputs=[])

    def _check_call(self, x: torch.Tensor, what: str, multiple: int):
        if x.ndim != 4 or x.shape[-2] % multiple or x.shape[-1] % multiple:
            raise ValueError(f"EDMAutoencoder.{what}: input of shape {tuple(x.shape)}; the GPU path takes [n, c, h, w] "
                             f"with h and w multiples of {multiple}")
        if self.config["direct_skips"]:
            raise NotImplementedError("direct_skips is not implemented by the GPU path (no shipped autoencoder uses it)")
        if self.training:
            raise L.TdxError("the GPU path is inference-only: call model.eval()")
        if x.device.type != "cuda":
            raise L.TdxError(f"EDMAutoencoder.{what} (GPU path) got a CPU tensor; there is no CPU fallback")

    def folded(self) -> FoldedWeights:
        """The decoder's folded weights (the encoder folds its own, EDMUnet2D.folded)."""
        if self._folded is None:
            dev = self.device
            if dev.type != "cuda":
                raise L.TdxError("EDMAutoencoder (GPU path) needs its parameters on a CUDA device; there is no CPU path")
            L.lib()
            self._folded = FoldedWeights(self.decoder_view(), dev, plan=autoencoder_decoder_plan(self._decoder_config()))
        return self._folded

    def decoder_view(self) -> SimpleNamespace:
        """The decoder named as FoldedWeights reads an EDMUnet2D: `decoder_conv` is the first convolution
        `enc.conv`, `decoder.{i}.` is `dec.{i}.` (block i of autoencoder_decoder_plan), out_conv / out_gain as they are."""
        sd = {}
        for k, v in self.state_dict().items():
            if k.startswith("decoder."):
                sd["dec." + k[len("decoder."):]] = v
            elif k == "decoder_conv.weight":
                sd["enc.conv.weight"] = v
            elif k in ("out_conv.weight", "out_gain"):
                sd[k] = v
        return SimpleNamespace(config=self._decoder_config(), state_dict=lambda: sd)

    def _decode_plan(self, n, h, w):
        key = ("dec", n, h, w)
        if key not in self._plans:
            fw = self.folded()
            dev = fw.device
            em = UNetEmitter(fw, n, h, w)
            bufs = SimpleNamespace(z=torch.zeros((n, fw.in_channels, h, w), dtype=torch.float32, device=dev),
                                   out=torch.zeros((n, fw.out_channels, em.out_h, em.out_w), dtype=torch.float32,
                                                   device=dev))
            prog = UNetProgram(dev)
            em.emit(prog, [(bufs.z, fw.in_channels, None)], model_out=bufs.out)
            self._plans[key] = (prog, bufs)
            while len(self._plans) > self.max_cached_plans:       # every plan owns a full activation arena + a graph
                self._plans.pop(next(iter(self._plans)))
        else:
            self._plans[key] = self._plans.pop(key)               # most recently used last
        return self._plans[key]

    @torch.no_grad()
    def preencode(self, x, conditional_inputs=None):
        """(means, logvars), each [n, latent_channels, h/8, w/8] for the shipped 4-level model."""
        self._check_call(x, "preencode", 8 * 2 ** (len(self.config["model_channel_mults"] or [1, 2, 3, 4]) - 1))
        self.encoder.use_cuda_graph = self.use_cuda_graph
        encodings = self.encoder(x, noise_labels=None, conditional_inputs=conditional_inputs)
        half = encodings.shape[1] // 2
        return encodings[:, :half], encodings[:, half:]

    def postencode(self, means, logvars, use_mode=False):
        if use_mode:
            return means
        std = torch.exp(logvars * 0.5)
        eps = torch.randn_like(std)
        return means + eps * std

    @torch.no_grad()
    def decode(self, z, include_logvar=False):
        self._check_call(z, "decode", 8)
        n, c, h, w = z.shape
        if c != self.config["latent_channels"]:
            raise ValueError(f"decode got {c} latent channels; the model has {self.config['latent_channels']}")
        prog, bufs = self._decode_plan(n, h, w)
        bufs.z.copy_(z)
        prog.run(self.use_cuda_graph)
        out = bufs.out.to(z.dtype, copy=True)
        if include_logvar:
            return out, self.logvar.reshape(-1, 1, 1, 1)
        return out

    def norm_weights(self):
        """Reference training hook; weights are re-normalised at fold time here."""
        return None
