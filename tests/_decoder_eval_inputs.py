"""Inputs of the decoder evaluations' golden (tests/golden/decoder_eval_golden.npz): the seeded stand-in for the drivers'
dataset (H5DecoderTerrainDataset batches through LongDataset: 'image', 'lowfreq_padded', 'cond_img'), the cases and the
drivers' batching.  Shared by tests/golden/make_golden_decoder_eval.py and the tests, so both see the same batches
without storing them."""
from __future__ import annotations

import hashlib

import numpy as np
import torch
import torch.nn.functional as F

RESIDUAL_MEAN, RESIDUAL_STD, SIGMA_DATA = 0.0, 1.1678, 0.5     # consistency_decoder_64-3.cfg [results_dataset]
DATASET_SEED, GENERATOR_SEED = 958, 548                        # the drivers' LongDataset seed and noise generator seed

# name: the driver, its options and what they make of the dataset (image size S, tiles T at stride, crop)
CASES = {
    "dc": dict(driver="decoder_consistency", size=128, tile_size=64, tile_stride=32, intermediate_sigma=0.065,
               num_images=2, batch_size=2, crop=None),
    "dc1": dict(driver="decoder_consistency", size=128, tile_size=64, tile_stride=32, intermediate_sigma=0.0,
                num_images=2, batch_size=2, crop=None),
    "dct": dict(driver="decoder_consistency", size=128, tile_size=64, tile_stride=32, intermediate_sigma=0.065,
                num_images=3, batch_size=2, crop=None),
    "tiled": dict(driver="tiled_decoder_consistency", size=896, tile_size=512, tile_stride=384,
                  intermediate_sigma=0.065, num_images=1, batch_size=1, crop=512),
}
# every stored terrain plane keeps rows and columns 0, k, 2k, ... (the full planes would make the fixture megabytes)
SUBSAMPLE = {"dc": 2, "dc1": 2, "dct": 2, "tiled": 4}


def dataset_item(index: int, size: int, seed: int = DATASET_SEED) -> dict:
    """Item `index` of the stand-in dataset at crop `size`: the normalised residual times sigma_data, the low-frequency
    plane with its one-pixel border (signed-sqrt metres) and four latent channels nearest-upsampled x8."""
    g = torch.Generator().manual_seed(seed * 100003 + index)
    h = size // 8
    image = torch.randn(1, size, size, generator=g) * SIGMA_DATA
    lowfreq_padded = torch.randn(1, h + 2, h + 2, generator=g) * 8.0 + 20.0
    latent = torch.randn(4, h, h, generator=g)
    cond_img = F.interpolate(latent[None], size=(size, size), mode="nearest")[0]
    return {"image": image, "lowfreq_padded": lowfreq_padded, "cond_img": cond_img}


def batches(case: str):
    """The batches a driver evaluates in `case`: batch_size consecutive dataset items, the last one truncated to the
    images still missing, as dicts of [b, ...] tensors."""
    c = CASES[case]
    done, index = 0, 0
    while done < c["num_images"]:
        items = [dataset_item(index + i, c["size"]) for i in range(c["batch_size"])]
        index += c["batch_size"]
        b = min(c["batch_size"], c["num_images"] - done)
        yield {k: torch.stack([it[k] for it in items])[:b] for k in items[0]}
        done += b


def digest(t) -> str:
    """sha256 of an array's bytes (fp32 planes too large to store are pinned bit for bit by their digest)."""
    a = np.ascontiguousarray(t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t)
    return hashlib.sha256(a.tobytes()).hexdigest()
