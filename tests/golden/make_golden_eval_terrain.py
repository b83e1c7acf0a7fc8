"""Generate tests/golden/eval_terrain_golden.npz: the evaluation drivers' terrain decode, `_decode_latents_to_terrain`
of the UNMODIFIED reference (evaluation/base_consistency.py:34-72, checkout at $TERRAIN_DIFFUSION_REF), fp32 and with
the decoder under the reference's own CPU bf16 autocast, on procedural decoder weights (oracle.unet.DECODER_CFG,
oracle.unet.procedural_state_dict seed 0, re-created identically in the tests).

    python tests/golden/make_golden_eval_terrain.py

The driver module itself imports the training stack (accelerate, torchmetrics, confection, h5py), so the function's
source is taken from it with `ast` and run with the reference's own laplacian_denoise / laplacian_decode and
sample_decoder_consistency_tiled, as the module binds them.  The dataset is a stand-in with the attributes and the
denormalize_residual / denormalize_lowfreq methods of H5LatentsDataset (training/datasets/h5_latents_dataset.py:
360-366); case "a" reaches it through `.base_dataset`, as the drivers' dataset wrappers do.

Cases (inputs are stored next to the outputs; the noise is torch.randn((B, 1, 8h, 8w), generator=CPU generator seeded
with <case>.noise_seed), the function's own draw):
  a   B=5, 8x8 latents,  inter_t [0.13] (two phases), denoising on
  b   B=2, 8x8 latents,  inter_t []     (one phase),  denoising off
  c   B=1, 8x16 latents, inter_t [0.13],              denoising off (two 64^2 tiles per image)
  d   B=2, 8x16 latents, inter_t [],                  denoising on
<case>.ref_bf16_err is rel-RMS(terrain with every decoder forward under CPU bf16 autocast, fp32 terrain): the
reference's own error when its model computes in bf16 (the read-out stays fp32, as in the drivers' decode).
"""
from __future__ import annotations

import ast
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]

from terrain_diffusion.data.laplacian_encoder import laplacian_decode, laplacian_denoise  # noqa: E402
from terrain_diffusion.models.edm_unet import EDMUnet2D  # noqa: E402
from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler  # noqa: E402
from terrain_diffusion.training.evaluation.sample_diffusion_decoder import sample_decoder_consistency_tiled  # noqa

from oracle import unet as O  # noqa: E402

torch.set_grad_enabled(False)

CASES = {   # name: (B, h, w, inter_t, disable_laplacian_denoising, through .base_dataset)
    "a": (5, 8, 8, [0.13], False, True),
    "b": (2, 8, 8, [], True, False),
    "c": (1, 8, 16, [0.13], True, False),
    "d": (2, 8, 16, [], False, False),
}
LATENTS_MEAN = [0.1, -0.2, 0.05, 0.3]
LATENTS_STD = [1.2, 0.8, 1.5, 0.9]
RESIDUAL_MEAN, RESIDUAL_STD = 0.25, 1.75


def reference_functions() -> dict:
    """_decode_latents_to_terrain and _normalize_uint8_three_channel from base_consistency.py, bound to the names the
    module imports them under."""
    path = REF / "terrain_diffusion" / "evaluation" / "base_consistency.py"
    tree = ast.parse(path.read_text())
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef)
            and n.name in ("_decode_latents_to_terrain", "_normalize_uint8_three_channel")]
    ns = {"torch": torch, "laplacian_denoise": laplacian_denoise, "laplacian_decode": laplacian_decode,
          "sample_decoder_consistency_tiled": sample_decoder_consistency_tiled}
    exec(compile(ast.Module(body=keep, type_ignores=[]), str(path), "exec"), ns)
    return ns


class LatentsStats:
    """The attributes and methods of H5LatentsDataset that the decode uses."""

    def __init__(self):
        self.latents_mean = torch.tensor(LATENTS_MEAN).view(1, 4, 1, 1)
        self.latents_std = torch.tensor(LATENTS_STD).view(1, 4, 1, 1)
        self.residual_mean, self.residual_std = RESIDUAL_MEAN, RESIDUAL_STD

    def denormalize_residual(self, residual):
        return residual * self.residual_std + self.residual_mean

    def denormalize_lowfreq(self, lowfreq):
        return lowfreq * 38.6 + -31.4


class Wrapped:
    def __init__(self, base):
        self.base_dataset = base


class Bf16Forward(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model
        self.config = model.config

    def forward(self, *args, **kwargs):
        with torch.autocast("cpu", dtype=torch.bfloat16):
            return self.model(*args, **kwargs)


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def samples_for(name, B, h, w):
    g = torch.Generator().manual_seed(100 + ord(name))
    s = torch.randn(B, 5, h, w, generator=g)
    s[:, 4] = s[:, 4] * 0.8 + 0.5       # the low-frequency channel: a few tens of signed-sqrt metres once de-normalised
    return s


def main():
    fns = reference_functions()
    decode = fns["_decode_latents_to_terrain"]
    dec = EDMUnet2D(**O.DECODER_CFG).eval()
    dec.load_state_dict(O.procedural_state_dict(O.DECODER_CFG, seed=0))
    dec16 = Bf16Forward(dec)
    out = {"latents_mean": np.array(LATENTS_MEAN, np.float32), "latents_std": np.array(LATENTS_STD, np.float32),
           "residual_mean": np.float64(RESIDUAL_MEAN), "residual_std": np.float64(RESIDUAL_STD)}
    for name, (B, h, w, inter_t, no_denoise, wrapped) in CASES.items():
        samples = samples_for(name, B, h, w)
        seed = 1000 + ord(name)
        ds = Wrapped(LatentsStats()) if wrapped else LatentsStats()

        def run(model):
            return decode(samples.clone(), ds, model, EDMDPMSolverMultistepScheduler(),
                          torch.Generator().manual_seed(seed), inter_t=inter_t,
                          disable_laplacian_denoising=no_denoise).float()
        t0 = time.time()
        y32 = run(dec)
        y16 = run(dec16)
        err = rel_rms(y16, y32)
        print(f"{name}: {tuple(y32.shape)}  {time.time() - t0:.0f}s  bf16 err {err:.4g}", flush=True)
        out.update({f"{name}.samples": samples.numpy(), f"{name}.noise_seed": np.int64(seed),
                    f"{name}.inter_t": np.array(inter_t, np.float64), f"{name}.denoise": np.bool_(not no_denoise),
                    f"{name}.wrapped": np.bool_(wrapped), f"{name}.y": y32.numpy(),
                    f"{name}.ref_bf16_err": np.float64(err)})
    images = torch.from_numpy(out["a.y"]) * 40.0
    out["uint8.images"] = images.numpy()
    out["uint8.y"] = fns["_normalize_uint8_three_channel"](images).numpy()
    np.savez_compressed(HERE / "eval_terrain_golden.npz", **out)
    print(f"wrote {len(out)} arrays, {os.path.getsize(HERE / 'eval_terrain_golden.npz') / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
