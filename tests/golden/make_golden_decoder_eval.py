"""Generate tests/golden/decoder_eval_golden.npz: the decoder evaluations of the UNMODIFIED reference
(evaluation/decoder_consistency.py and tiled_decoder_consistency.py, checkout at $TERRAIN_DIFFUSION_REF), run through
their click commands' `main.callback` on the CPU, fp32 and with the decoder under CPU bf16 autocast, on procedural
decoder weights (oracle.unet.DECODER_CFG, oracle.unet.procedural_state_dict seed 0, re-created identically in the tests).

    TERRAIN_DIFFUSION_REF=<checkout> python tests/golden/make_golden_decoder_eval.py

The drivers import the training stack, so stand-ins go into sys.modules first: `accelerate` (a CPU Accelerator whose
autocast() is off, or CPU bf16 autocast for the bf16 run), `confection` (Config().from_disk returns the [scheduler] and
[results_dataset] sections of consistency_decoder_64-3.cfg plus one section the driver deletes; registry.resolve
builds the scheduler), `torchmetrics` (FID / KID that record the uint8 images handed to update()), the training
registry, `LongDataset` (tests/_decoder_eval_inputs.dataset_item, read through the drivers' own DataLoader), and the
absent third-party modules the drivers' other imports need (`easydict`, `ema_pytorch`, `matplotlib`, no arithmetic).
`EDMUnet2D.from_pretrained` returns the procedural decoder.  The module global `laplacian_decode` of each driver is
wrapped to record its fp32 outputs; every other line runs as shipped.

Cases: tests/_decoder_eval_inputs.CASES.  Per case:
  <case>.t                   the fp32 noise labels the model sees, one per step
  <case>.<k>.fake / .real    batch k's terrain handed to the metric before the uint8 normalisation (laplacian_decode,
                             sign(x) x^2 and the crop, as the driver applies them), every SUBSAMPLE-th row and column
  <case>.<k>.fake_u8 / .real_u8   the uint8 images of image_metric.update(real=False / True), channel 0 (the driver
                             repeats it to three), subsampled likewise; <case>.<k>.u8_3ch says all three were equal
  dc.<k>.fake_ld_arg / .fake_ld   the residual argument (full) and the output (subsampled) of the generated image's
                             laplacian_decode in case dc
  <case>.ref_bf16_err        rel-RMS(generated terrain with the decoder under CPU bf16 autocast, fp32 run): the
                             reference's own error when its model computes in bf16
  <case>.ref_bf16_u8_diff    the largest |uint8 difference| between those two runs' generated images
window64 is `_get_weights(64)`; window_sha.<T> the sha256 of `_get_weights(T)` for T = 64, 128, 512.
"""
from __future__ import annotations

import contextlib
import os
import sys
import time
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF = Path(os.environ["TERRAIN_DIFFUSION_REF"])   # a checkout of the original terrain-diffusion project
sys.path[:0] = [str(ROOT / "oracle" / "_stub"), str(REF), str(ROOT)]

from oracle import unet as O  # noqa: E402
from tests import _decoder_eval_inputs as I  # noqa: E402

torch.set_grad_enabled(False)
BF16 = [False]          # the bf16 run: the stand-in Accelerator's autocast() enters CPU bf16 autocast
UPDATES: list = []      # (real, uint8 images) of every image_metric.update
DECODES: list = []      # every laplacian_decode output
LABELS: list = []       # the noise labels of every model call


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class Accelerator:
    def __init__(self, mixed_precision=None):
        self.device = torch.device("cpu")

    def prepare(self, model):
        return model

    def autocast(self):
        return torch.autocast("cpu", dtype=torch.bfloat16) if BF16[0] else contextlib.nullcontext()


CONFIG = {"trainer": {"@trainer": "consistency"},
          "scheduler": {"@scheduler": "edm_dpm", "sigma_min": 0.002, "sigma_max": 80, "sigma_data": 0.5},
          "results_dataset": {"@dataset": "h5_decoder_terrain", "crop_size": 512, "residual_mean": I.RESIDUAL_MEAN,
                              "residual_std": I.RESIDUAL_STD, "sigma_data": I.SIGMA_DATA}}


class Config(dict):
    def from_disk(self, path):
        return Config({k: dict(v) for k, v in CONFIG.items()})


class Registry:
    @staticmethod
    def resolve(config, validate=True):
        from terrain_diffusion.scheduler.dpmsolver import EDMDPMSolverMultistepScheduler
        sch = {k: v for k, v in config["scheduler"].items() if not k.startswith("@")}
        return {"scheduler": EDMDPMSolverMultistepScheduler(**sch), "results_dataset": dict(config["results_dataset"])}


class Metric:
    def __init__(self, normalize=False):
        pass

    def to(self, device):
        return self

    def update(self, images, real):
        UPDATES.append((bool(real), images.clone()))

    def compute(self):
        return torch.tensor(0.0)


class LongDataset(torch.utils.data.Dataset):
    def __init__(self, base_dataset, length=10 ** 12, shuffle=True, seed=None):
        self.size = int(base_dataset["crop_size"])
        self.length = length

    def __len__(self):
        return self.length

    def __getitem__(self, index):
        return I.dataset_item(index, self.size)


def install_stand_ins():
    _module("accelerate", Accelerator=Accelerator)
    _module("confection", Config=Config, registry=Registry())
    _module("torchmetrics")
    _module("torchmetrics.image")
    _module("torchmetrics.image.fid", FrechetInceptionDistance=Metric)
    _module("torchmetrics.image.kid", KernelInceptionDistance=Metric)
    _module("easydict", EasyDict=dict)
    _module("ema_pytorch", PostHocEMA=object)
    _module("matplotlib")
    _module("matplotlib.pyplot")
    _module("terrain_diffusion.training.registry", build_registry=lambda: None)
    _module("terrain_diffusion.training.datasets", LongDataset=LongDataset)
    from terrain_diffusion.models.edm_unet import EDMUnet2D

    def from_pretrained(cls, path, **kw):
        m = EDMUnet2D(**O.DECODER_CFG).eval()
        m.load_state_dict(O.procedural_state_dict(O.DECODER_CFG, seed=0))
        m.register_forward_pre_hook(lambda mod, args, kwargs: LABELS.append(kwargs["noise_labels"].clone()),
                                    with_kwargs=True)
        return m
    EDMUnet2D.from_pretrained = classmethod(from_pretrained)


def run_driver(mod, c, bf16):
    BF16[0] = bf16
    UPDATES.clear(), DECODES.clear(), LABELS.clear()
    kw = dict(model_path=None, config_path="consistency_decoder_64-3.cfg", num_images=c["num_images"],
              batch_size=c["batch_size"], intermediate_sigma=c["intermediate_sigma"], metric="fid", save_images=0,
              experiment_name="golden")
    if c["driver"] == "decoder_consistency":
        kw.update(tile_size=c["tile_size"], tile_stride=c["tile_stride"], image_size=c["size"])
    else:
        assert (c["size"], c["tile_size"], c["tile_stride"], c["crop"]) == (896, 512, 384, 512)
    mod.main.callback(**kw)
    return list(UPDATES), list(DECODES), list(LABELS)


def terrain(ld_out, crop):
    """The driver's two lines between laplacian_decode and the metric: sign(x) x^2, then the centre crop."""
    t = torch.sign(ld_out) * torch.square(ld_out)
    if crop:
        s = (t.shape[-1] - crop) // 2
        t = t[..., s:s + crop, s:s + crop]
    return t


def rel_rms(a, b):
    return float((a - b).square().mean().sqrt() / (b.square().mean().sqrt() + 1e-30))


def main():
    install_stand_ins()
    import importlib
    mods = {}
    for name in ("decoder_consistency", "tiled_decoder_consistency"):
        mod = importlib.import_module(f"terrain_diffusion.evaluation.{name}")
        original = mod.laplacian_decode

        def recording(*args, _f=original, **kwargs):
            out = _f(*args, **kwargs)
            DECODES.append((args[0].clone(), out.clone()))
            return out
        mod.laplacian_decode = recording
        mods[name] = mod
    get_weights = mods["decoder_consistency"]._get_weights
    out = {"window64": get_weights(64)[0, 0].numpy()}
    for T in (64, 128, 512):
        out[f"window_sha.{T}"] = np.str_(I.digest(get_weights(T)[0, 0]))
    for name, c in I.CASES.items():
        t0 = time.time()
        k_sub = I.SUBSAMPLE[name]
        upd, dec, labels = run_driver(mods[c["driver"]], c, bf16=False)
        upd16, dec16, _ = run_driver(mods[c["driver"]], c, bf16=True)
        n_steps = 2 if c["intermediate_sigma"] > 0 else 1
        out[f"{name}.t"] = np.array([float(lab[0]) for lab in labels[:n_steps]], np.float32)
        assert all(lab.dtype == torch.float32 for lab in labels)
        n_batches = len(dec) // 2
        assert len(upd) == len(dec) == len(dec16) == 2 * n_batches
        fakes, fakes16, u8_diff = [], [], 0
        for k in range(n_batches):
            (_, fake_u8), (_, real_u8) = upd[2 * k], upd[2 * k + 1]
            assert not upd[2 * k][0] and upd[2 * k + 1][0]
            (fake_arg, fake_ld), (_, real_ld) = dec[2 * k], dec[2 * k + 1]
            fake, real = terrain(fake_ld, c["crop"]), terrain(real_ld, c["crop"])
            fakes.append(fake)
            fakes16.append(terrain(dec16[2 * k][1], c["crop"]))
            u8_diff = max(u8_diff, int((upd16[2 * k][1].int() - fake_u8.int()).abs().max()))
            sub = (slice(None), 0, slice(None, None, k_sub), slice(None, None, k_sub))
            out.update({f"{name}.{k}.fake": fake[sub].numpy(), f"{name}.{k}.real": real[sub].numpy(),
                        f"{name}.{k}.fake_u8": fake_u8[sub].numpy(), f"{name}.{k}.real_u8": real_u8[sub].numpy(),
                        f"{name}.{k}.u8_3ch": np.bool_(all(torch.equal(u[:, 0], u[:, i]) for u in (fake_u8, real_u8)
                                                           for i in (1, 2)))})
            if name == "dc":
                out[f"{name}.{k}.fake_ld_arg"] = fake_arg.numpy()
                out[f"{name}.{k}.fake_ld"] = fake_ld[sub].numpy()
        err = rel_rms(torch.cat(fakes16), torch.cat(fakes))
        out[f"{name}.ref_bf16_err"] = np.float64(err)
        out[f"{name}.ref_bf16_u8_diff"] = np.int64(u8_diff)
        out[f"{name}.batches"] = np.int64(n_batches)
        print(f"{name}: {n_batches} batches, t {out[f'{name}.t']}, {time.time() - t0:.0f}s, bf16 err {err:.4g}, "
              f"uint8 diff {u8_diff}", flush=True)
    np.savez_compressed(HERE / "decoder_eval_golden.npz", **out)
    print(f"wrote {len(out)} arrays, {os.path.getsize(HERE / 'decoder_eval_golden.npz') / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
