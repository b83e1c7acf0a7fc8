"""Generate tests/golden/autoencoder_golden.npz: EDMAutoencoder.preencode / decode and the two tiled samplers of
training/evaluation/sample_autoencoder.py from the UNMODIFIED reference (checkout at $TERRAIN_DIFFUSION_REF), fp32
and the reference's own CPU bf16 autocast, on the x8 architecture (oracle.autoencoder.X8_CFG) with procedural
weights (oracle.autoencoder.procedural_state_dict, seed 0, re-created identically in the tests).

    python tests/golden/make_golden_autoencoder.py

Cases (inputs are stored next to the outputs):
  enc    preencode, B=2, 64^2 images                            -> <case>.means, <case>.logvars
  dec    decode, B=2, 8^2 latents                               -> <case>.y
  rec96  sample_autoencoder_tiled(use_mode=True), 1x1x96^2, tile 64, stride 32 (2x2 tiles)
  dec96  decode_autoencoder_latents_tiled, 1x4x12^2 latents (96^2 out), tile 64, stride 32
<case>.ref_bf16_err is rel-RMS(bf16 output, fp32 output) of the reference itself (for enc: of [means, logvars]).
shapes.<x8|lpbd3>.names / .shapes: the reference class's state-dict entries for X8_CFG and for X8_CFG with
layers_per_block_decoder=3 (shapes as "-"-joined strings, "" for a scalar).
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]

from terrain_diffusion.models.edm_autoencoder import EDMAutoencoder  # noqa: E402
from terrain_diffusion.training.evaluation.sample_autoencoder import (  # noqa: E402
    decode_autoencoder_latents_tiled, sample_autoencoder_tiled)

from oracle import autoencoder as OA  # noqa: E402

torch.set_grad_enabled(False)


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def both(fn):
    """fp32 output and the reference's own bf16 output of the same call (CPU bf16 autocast)."""
    y32 = fn().float()
    with torch.autocast("cpu", dtype=torch.bfloat16):
        y16 = fn().float()
    print(f"  bf16 err {rel_rms(y16, y32):.4g}", flush=True)
    return y32, y16


def inputs():
    g = torch.Generator().manual_seed(21)
    x = torch.randn(2, 1, 64, 64, generator=g)
    z = torch.randn(2, 4, 8, 8, generator=g)
    img96 = torch.randn(1, 1, 96, 96, generator=g)
    lat12 = torch.randn(1, 4, 12, 12, generator=g)
    return x, z, img96, lat12


def main():
    out = {}
    for tag, extra in (("x8", {}), ("lpbd3", {"layers_per_block_decoder": 3})):
        sd = EDMAutoencoder(**OA.X8_CFG, **extra).state_dict()
        out[f"shapes.{tag}.names"] = np.array(list(sd))
        out[f"shapes.{tag}.shapes"] = np.array(["-".join(map(str, v.shape)) for v in sd.values()])
    model = EDMAutoencoder(**OA.X8_CFG).eval()
    model.load_state_dict(OA.procedural_state_dict(OA.X8_CFG, seed=0))
    x, z, img96, lat12 = inputs()
    out.update({"enc.x": x.numpy(), "dec.z": z.numpy(), "rec96.images": img96.numpy(), "dec96.latents": lat12.numpy()})

    print("enc", flush=True)
    y32, y16 = both(lambda: torch.cat(model.preencode(x), dim=1))
    out["enc.means"], out["enc.logvars"] = y32[:, :4].numpy(), y32[:, 4:].numpy()
    out["enc.ref_bf16_err"] = np.float64(rel_rms(y16, y32))
    for case, fn in (("dec", lambda: model.decode(z)),
                     ("rec96", lambda: sample_autoencoder_tiled(model, img96, 64, 32, use_mode=True)),
                     ("dec96", lambda: decode_autoencoder_latents_tiled(model, lat12, 64, 32))):
        print(case, flush=True)
        y32, y16 = both(fn)
        out[f"{case}.y"], out[f"{case}.ref_bf16_err"] = y32.numpy(), np.float64(rel_rms(y16, y32))
    np.savez_compressed(HERE / "autoencoder_golden.npz", **out)
    print(f"wrote {len(out)} arrays, {os.path.getsize(HERE / 'autoencoder_golden.npz') / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
