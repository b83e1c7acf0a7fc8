"""ORACLE (test infrastructure, not product): CPU fp32 restatement of the reference's EDM autoencoder and its tiled
evaluation samplers (xandergos/terrain-diffusion @ 82a0431):

  EDMAutoencoder.__init__ (decoder plan) / preencode / decode    terrain_diffusion/models/edm_autoencoder.py:13-158
  sample_autoencoder_tiled / decode_autoencoder_latents_tiled    terrain_diffusion/training/evaluation/
                                                                 sample_autoencoder.py:8-119

The encoder is the encode_only EDMUnet2D of oracle/unet.py; the decoder blocks are oracle.unet.unet_block.  Parity
pinned: tests/test_autoencoder_cpu.py checks this file against tests/golden/autoencoder_golden.npz, written from the
unmodified reference by tests/golden/make_golden_autoencoder.py.  direct_skips is not restated (no shipped model uses it).
"""
from __future__ import annotations

import math

import torch

from . import tiling as otile
from . import unet as ounet

X8_CFG = dict(image_size=512, in_channels=1, out_channels=1, model_channels=64, model_channel_mults=[1, 2, 4, 4],
              layers_per_block=2, attn_resolutions=[], midblock_attention=False, latent_channels=4,
              conditional_inputs=[], direct_skips=[])
"""configs/autoencoder/autoencoder_x8.cfg [model] (the model block of autoencoder_x8_squared.cfg is the same); keys
the reference's constructor does not take (emb_channels, noise_emb_dims, ...) are left out."""


def encoder_config(cfg: dict) -> dict:
    """The encoder's EDMUnet2D arguments (edm_autoencoder.py:67-84)."""
    return dict(image_size=cfg["image_size"], in_channels=cfg["in_channels"], out_channels=cfg["latent_channels"] * 2,
                model_channels=cfg.get("model_channels", 128), model_channel_mults=cfg.get("model_channel_mults"),
                layers_per_block=cfg.get("layers_per_block", 3), emb_channels=0, noise_emb_dims=0,
                attn_resolutions=cfg.get("attn_resolutions"), midblock_attention=cfg.get("midblock_attention", True),
                logvar_channels=cfg.get("logvar_channels", 128), block_kwargs=cfg.get("block_kwargs"),
                conditional_inputs=cfg.get("conditional_inputs") or [], encode_only=True)


def decoder_plan(cfg: dict) -> list:
    """The `decoder` ModuleList (edm_autoencoder.py:86-103) as oracle.unet block dicts."""
    mults = cfg.get("model_channel_mults") or [1, 2, 3, 4]
    mc = cfg.get("model_channels", 128)
    lpb = cfg.get("layers_per_block_decoder") or cfg.get("layers_per_block", 3)
    if isinstance(lpb, int):
        lpb = [lpb] * len(mults)
    attn_res = cfg.get("attn_resolutions") or []
    cout = mc * mults[-1]
    blocks = []
    for level, (channels, nb) in reversed(list(enumerate(zip([mc * m for m in mults], lpb)))):
        res = cfg["image_size"] // 2 ** level
        if level == len(mults) - 1:
            blocks.append(dict(mode="dec", resample="keep", cin=cout, cout=cout,
                               attention=cfg.get("midblock_attention", True)))
            blocks.append(dict(mode="dec", resample="keep", cin=cout, cout=cout, attention=False))
        else:
            blocks.append(dict(mode="dec", resample="up", cin=cout, cout=cout, attention=False))
        for _ in range(nb + 1):
            blocks.append(dict(mode="dec", resample="keep", cin=cout, cout=channels, attention=res in attn_res))
            cout = channels
    return blocks


def state_shapes(cfg: dict) -> dict:
    """Parameter / buffer names and shapes of the reference EDMAutoencoder."""
    shapes = {"out_gain": (), "logvar": (cfg.get("n_logvar", 1),)}
    no_emb = not cfg.get("conditional_inputs")          # noise_emb_dims=0 and no conditions: emb_channels = 0
    shapes.update({"encoder." + k: v for k, v in ounet.state_shapes(encoder_config(cfg)).items()
                   if not (no_emb and k.endswith(".emb_linear.weight"))})
    cph = (cfg.get("block_kwargs") or {}).get("channels_per_head", 64)
    for i, b in enumerate(decoder_plan(cfg)):
        p = f"decoder.{i}."
        shapes[p + "emb_gain"] = ()
        shapes[p + "conv_res0.weight"] = (b["cout"], b["cin"], 3, 3)
        shapes[p + "conv_res1.weight"] = (b["cout"], b["cout"], 3, 3)
        if b["cin"] != b["cout"]:
            shapes[p + "conv_skip.weight"] = (b["cout"], b["cin"], 1, 1)
        if b["attention"] and b["cout"] // cph:
            shapes[p + "attn_qkv.weight"] = (b["cout"] * 3, b["cout"], 1, 1)
            shapes[p + "attn_proj.weight"] = (b["cout"], b["cout"], 1, 1)
    mults = cfg.get("model_channel_mults") or [1, 2, 3, 4]
    mc = cfg.get("model_channels", 128)
    shapes["decoder_conv.weight"] = (mc * mults[-1], cfg["latent_channels"] + len(cfg.get("direct_skips") or []) + 1,
                                     1, 1)
    shapes["out_conv.weight"] = (cfg.get("out_channels") or cfg["in_channels"], mc * mults[0], 3, 3)
    return shapes


def procedural_state_dict(cfg: dict, seed: int = 0) -> dict:
    """oracle.unet.procedural_state_dict's per-name draws for every tensor; the gains keep the reference's
    initial values (encoder.out_gain 1, out_gain 0.1, emb_gain unused without an embedding), which are non-zero."""
    import zlib
    sd = {}
    for name, shape in state_shapes(cfg).items():
        g = torch.Generator().manual_seed((zlib.crc32(name.encode()) ^ seed) & 0x7FFFFFFF)
        if name == "encoder.out_gain":
            sd[name] = torch.ones([])
        elif name == "out_gain":
            sd[name] = torch.ones([]) * 0.1
        elif name.endswith("emb_gain") or name == "logvar":
            sd[name] = torch.zeros(shape)
        elif name.endswith(".freqs"):
            sd[name] = 2 * math.pi * torch.randn(shape, generator=g)
        elif name.endswith(".phases"):
            sd[name] = 2 * math.pi * torch.rand(shape, generator=g)
        else:
            sd[name] = torch.randn(shape, generator=g)
    return sd


def _sub(sd: dict, prefix: str) -> dict:
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


@torch.no_grad()
def preencode(sd: dict, cfg: dict, x: torch.Tensor, conditional_inputs=None):
    """EDMAutoencoder.preencode (edm_autoencoder.py:107-123) without direct_skips: (means, logvars)."""
    enc = ounet.unet_forward(_sub(sd, "encoder."), encoder_config(cfg), x, None, conditional_inputs)
    half = enc.shape[1] // 2
    return enc[:, :half], enc[:, half:]


@torch.no_grad()
def decode(sd: dict, cfg: dict, z: torch.Tensor) -> torch.Tensor:
    """EDMAutoencoder.decode (edm_autoencoder.py:132-158) without direct_skips and logvar."""
    bk = cfg.get("block_kwargs") or {}
    kw = dict(res_balance=bk.get("res_balance", 0.3), attn_balance=bk.get("attn_balance", 0.3),
              clip_act=bk.get("clip_act", 256.0), channels_per_head=bk.get("channels_per_head", 64))
    x = ounet.mp_conv(torch.cat([z, torch.ones_like(z[:, :1])], dim=1), sd["decoder_conv.weight"])
    for i, b in enumerate(decoder_plan(cfg)):
        x = ounet.unet_block(x, None, sd, f"decoder.{i}.", b, **kw)
    return ounet.mp_conv(x, sd["out_conv.weight"], gain=sd["out_gain"])


@torch.no_grad()
def sample_autoencoder_tiled(sd, cfg, images, tile_size=None, tile_stride=None, *, eps=None):
    """sample_autoencoder_tiled (sample_autoencoder.py:8-58) with the linear window; eps: None for use_mode=True,
    else the list of per-tile unit draws in row-major tile order."""
    b, _, h, w = images.shape
    tile_size = tile_size or w
    tile_stride = tile_stride or tile_size
    weights = otile.linear_weight_window(tile_size)
    out_ch = cfg.get("out_channels") or cfg["in_channels"]
    output = torch.zeros((b, out_ch, h, w))
    output_w = torch.zeros_like(output)
    k = 0
    for i0 in otile.tile_starts(h, tile_size, tile_stride):
        for j0 in otile.tile_starts(w, tile_size, tile_stride):
            means, logvars = preencode(sd, cfg, images[..., i0:i0 + tile_size, j0:j0 + tile_size])
            latent = means if eps is None else means + eps[k] * torch.exp(logvars * 0.5)
            k += 1
            tile_out = decode(sd, cfg, latent)
            output[..., i0:i0 + tile_size, j0:j0 + tile_size] += tile_out * weights
            output_w[..., i0:i0 + tile_size, j0:j0 + tile_size] += weights
    return output / output_w


@torch.no_grad()
def decode_autoencoder_latents_tiled(sd, cfg, latents, tile_size=None, tile_stride=None):
    """decode_autoencoder_latents_tiled (sample_autoencoder.py:61-119) with the linear window."""
    b, _, lh, lw = latents.shape
    if tile_size is None:
        return decode(sd, cfg, latents)
    tile_stride = tile_stride or tile_size
    weights = otile.linear_weight_window(tile_size)
    out_h, out_w = lh * 8, lw * 8
    out_ch = cfg.get("out_channels") or cfg["in_channels"]
    output = torch.zeros((b, out_ch, out_h, out_w))
    output_w = torch.zeros_like(output)
    n_lat = math.ceil(tile_size / 8)
    for i0 in otile.tile_starts(out_h, tile_size, tile_stride):
        for j0 in otile.tile_starts(out_w, tile_size, tile_stride):
            li0, lj0 = i0 // 8, j0 // 8
            tile_out = decode(sd, cfg, latents[..., li0:min(lh, li0 + n_lat), lj0:min(lw, lj0 + n_lat)])
            io, jo = i0 - li0 * 8, j0 - lj0 * 8
            output[..., i0:i0 + tile_size, j0:j0 + tile_size] += \
                tile_out[..., io:io + tile_size, jo:jo + tile_size] * weights
            output_w[..., i0:i0 + tile_size, j0:j0 + tile_size] += weights
    return output / output_w
