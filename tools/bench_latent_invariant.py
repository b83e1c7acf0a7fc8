#!/usr/bin/env python
"""Cost of the batch-invariant latent stage on one GPU, with the shipped base architecture (procedural weights), the
shipped coarse and decoder architectures and a seeded `conditioning_fn`.

    python tools/bench_latent_invariant.py [--iters 10] [--repeats 5] [--out FILE]

It prints one JSON line, with the card's name, its enforced power limit and its SM clocks read in the same run, and
writes it to --out (default profiles/bench_latent_invariant.json):
  plans   the base forward's implicit-GEMM launches at 64^2 planned at one image and at 16 (the H100's plans): how many
          are split-K (at 16 images a split-K launch may be issued over image ranges), and how many launches of the
          anchored program at 16 images differ from the free plan there.
  stage   per tile-phase cost of `latent_stage_tiles` at n = 1, 2, 4, 8, 16 tiles per call, both phases, for the
          default path (pad_batch_to=16), the batch-invariant path anchored at 16 and the one anchored at 1: host wall
          time to a device synchronise over `iters` calls, median of `repeats`, the arms alternated.  Also the largest
          absolute difference and the rel-RMS of the invariant tiles against the default ones, and whether every
          invariant tile equals its one-tile call bit for bit.
  world   a cold 1024^2 `get()` and a cold `world.latents` read of the same area, latents_batch_invariant off and on
          (anchored at 16 and at 1), coarse_batch_size=16 and decoder_batch_size=4 in every arm; alternated, every
          cache emptied before each timed read.
Plans and graphs are built by warm-up calls first.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import math
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SIZES = (1, 2, 4, 8, 16)


def gpu_query(index: int) -> dict:
    """Enforced power limit (W) and SM clocks (MHz: current, maximum), read-only nvidia-smi queries."""
    out = {"power_limit_w": None, "sm_clock_mhz": None, "sm_clock_max_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        lim, sm, smax = (float(v) for v in q.stdout.strip().split(","))
        out.update(power_limit_w=lim, sm_clock_mhz=sm, sm_clock_max_mhz=smax)
    except Exception:
        pass
    return out


def wall(fn, sync) -> float:
    t0 = time.perf_counter()
    fn()
    sync()
    return time.perf_counter() - t0


def run(args):
    import torch

    from oracle import unet as ounet
    from terrain_diffusion_b200 import _lib as L
    from terrain_diffusion_b200.inference import WorldPipeline, pipeline, stages
    from terrain_diffusion_b200.inference.tiling import linear_weight_window
    from terrain_diffusion_b200.models import EDMUnet2D
    from tests._capture import RecordingEmitter, RecordingProgram, folded
    from tests.test_oracle_golden import BASE_CFG, COARSE_CFG
    if not torch.cuda.is_available():
        raise SystemExit("bench_latent_invariant.py measures the GPU path and needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    sync = torch.cuda.synchronize
    real_anchor = stages.latent_plan_images

    @contextlib.contextmanager
    def anchor(k):
        """The invariant path planned at k images (k None: the package's own choice)."""
        stages.latent_plan_images = real_anchor if k is None else (lambda top: k)
        pipeline.latent_plan_images = stages.latent_plan_images
        try:
            yield
        finally:
            stages.latent_plan_images = pipeline.latent_plan_images = real_anchor

    def build(cfg):
        m = EDMUnet2D(**cfg).eval()
        m.load_state_dict(ounet.procedural_state_dict(cfg, seed=0))
        return m.to(dev)

    def cond_fn(i1, i2, j1, j2):
        gg = torch.Generator().manual_seed((i1 * 7919 + j1 + 12345) & 0x7FFFFFFF)
        return torch.randn(5, i2 - i1, j2 - j1, generator=gg)

    coarse, base, dec = build(COARSE_CFG), build(BASE_CFG), build(ounet.DECODER_CFG)

    # ---------------- (a) the plans at each anchor
    def recorded(n, inv, k):
        fw = folded("base")
        prog = RecordingProgram()
        em = RecordingEmitter(fw, n, 64, 64, prog)
        em.batch_invariant, em.plan_images = inv, k
        meta = torch.device("meta")
        em.emit_embed(prog, emb_in=torch.empty((n, fw.emb_channels), device=meta))
        em.emit(prog, [(torch.empty((n, fw.in_channels, 64, 64), device=meta), fw.in_channels, None)],
                model_out=torch.empty((n, fw.out_channels, 64, 64), device=meta))
        return prog.igemm()

    plans = {}
    for k in (1, 16):
        shapes = [L.igemm_launch_shape(d) for d in recorded(k, False, 1)]
        split = [s for s in shapes if s[1] > 1]
        # a forced split-K launch holds one item per CTA: at 16 images it is issued as consecutive launches over image
        # ranges when its items do not fit the device at once (igemm_launch), so these are the candidates
        plans[str(k)] = {"igemm_launches": len(shapes), "split_k": len(split),
                         "split_k_shapes": sorted({f"N{n}xK{s}" for n, s in split}),
                         "differs_from_free_plan_at_16": sum(
                             (int(d.n_per_item), int(d.ksplit)) != L.igemm_launch_shape(f)
                             for d, f in zip(recorded(16, True, k), recorded(16, False, 1)))}

    # ---------------- (b) the stage
    ww = linear_weight_window(64, dev)
    g = torch.Generator().manual_seed(5)
    means, stds = torch.tensor(pipeline.COND_INPUT_MEAN), torch.tensor(pipeline.COND_INPUT_STD)
    hist = torch.zeros(1, 5)
    ctxs = [(0, i, j) for i in range(-2, 2) for j in range(-2, 2)]
    conds = []
    for _ in ctxs:
        w = torch.rand(1, 4, 4, generator=g) + 0.3
        v = means[:6].view(6, 1, 1) + stds[:6].view(6, 1, 1) * torch.randn(6, 4, 4, generator=g)
        conds.append(torch.cat([v * w, w]).to(dev))
    prevs = []
    for _ in ctxs:
        p = torch.randn(6, 64, 64, generator=g) * 0.6
        p[5] = torch.rand(64, 64, generator=g) + 0.5
        p[:5] *= p[5:]
        prevs.append(p.to(dev))
    t_init, t_inter = math.atan(80.0 / 0.5), math.atan(0.35 / 0.5)

    def stage(n, phase, inv):
        t, off, prev = (t_init, 5819, None) if phase == 1 else (t_inter, 5820, prevs[:n])
        return stages.latent_stage_tiles(base, 42, ctxs[:n], prev, conds[:n], t, ww, hist, means, stds,
                                         seed_offset=off, pad_batch_to=16, batch_invariant=inv)

    arms = {"default": (False, None), "invariant_anchor16": (True, 16), "invariant_anchor1": (True, 1)}
    diffs, identical = {}, {}
    for name, (inv, k) in arms.items():
        with anchor(k):
            for n in SIZES:
                for phase in (1, 2):
                    stage(n, phase, inv)               # warm-up: every program of every shape
    for name, (inv, k) in arms.items():
        if not inv:
            continue
        with anchor(k):
            ok, worst, num, den = True, 0.0, 0.0, 0.0
            for phase in (1, 2):
                ref = torch.stack(stage(16, phase, False)).double()
                got = torch.stack(stage(16, phase, True))
                for i in range(16):
                    one = stages.latent_stage_tiles(
                        base, 42, [ctxs[i]], None if phase == 1 else [prevs[i]], [conds[i]],
                        t_init if phase == 1 else t_inter, ww, hist, means, stds,
                        seed_offset=5819 if phase == 1 else 5820, pad_batch_to=16, batch_invariant=True)[0]
                    ok &= torch.equal(one.view(torch.int32), got[i].view(torch.int32))
                d = got.double()[:, :5] - ref[:, :5]
                worst = max(worst, float(d.abs().max()))
                num += float(d.square().sum())
                den += float(ref[:, :5].square().sum())
            identical[name] = bool(ok)
            diffs[name] = {"max_abs_diff": worst, "rel_rms": math.sqrt(num / den)}
    times = {(a, n): [] for a in arms for n in SIZES}
    for _ in range(args.repeats):
        for n in SIZES:
            for name, (inv, k) in arms.items():
                with anchor(k):
                    t = wall(lambda: [stage(n, p, inv) for _ in range(args.iters) for p in (1, 2)], sync)
                times[(name, n)].append(t / (args.iters * 2 * n))
    stage_rows = {name: {str(n): statistics.median(times[(name, n)]) * 1e3 for n in SIZES} for name in arms}

    # ---------------- (c) cold reads of a world
    def world(inv):
        w = WorldPipeline.from_local_models(coarse, base, dec, seed=42, cache_limit=None, conditioning_fn=cond_fn,
                                            coarse_batch_size=16, decoder_batch_size=4, latents_batch_invariant=inv,
                                            residual_mean=0.1, residual_std=1.2).to(dev).bind()
        return w

    reads = {"get_1024": lambda w: w.get(0, 0, 1024, 1024, with_climate=True),
             "latents_1024": lambda w: w.latents[:, 0:128, 0:128]}
    ws = {name: (world(inv), k) for name, (inv, k) in arms.items()}
    for name, (w, k) in ws.items():                  # warm-up: plans and graphs of every padded size
        with anchor(k):
            w.get(100_000, 100_000, 101_024, 101_024)
            w.latents[:, 20_000:20_128, 20_000:20_128]
    sync()
    res = {(r, a): [] for r in reads for a in ws}
    for _ in range(args.repeats):
        for r, read in reads.items():
            for name, (w, k) in ws.items():
                with anchor(k):
                    w.empty_cache()
                    t = time.perf_counter()
                    read(w)
                    sync()
                    res[(r, name)].append(time.perf_counter() - t)
    world_rows = [{"read": r, "arm": a, "wall_s": statistics.median(res[(r, a)]), "all_wall_s": res[(r, a)]}
                  for r in reads for a in ws]

    line = {"metric": "latents_batch_invariant: batch-invariant latent-stage solves at two plan anchors, cold reads",
            "plans_64": plans,
            "stage": {"ms_per_tile_phase": stage_rows, "iters": args.iters, "repeats": args.repeats,
                      "invariant_vs_default_n16": diffs, "invariant_bit_identical_to_one_tile": identical},
            "world": {"reads": {"get_1024": "world.get(0, 0, 1024, 1024, with_climate=True)",
                                "latents_1024": "world.latents[:, 0:128, 0:128]"},
                      "coarse_batch_size": 16, "decoder_batch_size": 4, "results": world_rows},
            "gpu": {"name": torch.cuda.get_device_name(dev), **gpu_query(dev.index)},
            "host": {"cores": len(os.sched_getaffinity(0))}, "torch": torch.__version__}
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=10, help="timed stage calls per repeat, arm and phase")
    ap.add_argument("--repeats", type=int, default=5, help="repeats (median) of every timed measurement")
    ap.add_argument("--out", default=str(ROOT / "profiles" / "bench_latent_invariant.json"),
                    help="write the JSON line here as well (default profiles/bench_latent_invariant.json)")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
