"""Measure the best (n_per_item, k_split) of every implicit-GEMM launch shape of the shipped models on THIS GPU and
write terrain_diffusion_b200/tuned_shapes.json (the planner's lookup table; the library's cost model is the fallback).

    python tools/tune_igemm.py [decoder|coarse|base ...]      # on the GPU; merges into the existing table

Method ("in the graph"): for one (model, batch, size) the whole forward is planned and replayed as its CUDA graph; then,
shape by shape in program order, every valid (N, k_split) of that shape is tried -- the forward is re-planned with the
candidate and the graph replay is timed (median of 3 x 20 replays) -- and the fastest is kept (coordinate descent, one
pass).  Timing the layer inside the real forward matters: back-to-back launches of one layer keep its weights and inputs
hot in L2 and favour weight-streaming shapes that lose inside the forward.
"""
import json
import os
import sys

os.environ["TDX_AUTOTUNE"] = "2"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from oracle import unet as O
from terrain_diffusion_b200.models import EDMUnet2D, plan
from tests.test_oracle_golden import BASE_CFG, COARSE_CFG


def time_forward(m, x, t, ci, reps=20):
    m._plans = {}
    m(x, t, ci)                      # plan + capture with the current table
    torch.cuda.synchronize()
    ts = []
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            m(x, t, ci)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / reps)
    return sorted(ts)[1]


def run(cfg, cases, cond=None):
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(O.procedural_state_dict(cfg, seed=0))
    m = m.cuda()
    table = plan.tuned_shapes()
    for n, hw in cases:
        x = torch.randn(n, cfg["in_channels"], hw, hw, device="cuda")
        t = torch.full((n,), 1.1, device="cuda")
        ci = cond(n) if cond else []
        plan._TUNE_CANDIDATES.clear()
        base = time_forward(m, x, t, ci)
        start = base
        keys = list(plan._TUNE_CANDIDATES.keys())
        for key in keys:
            cands = plan._TUNE_CANDIDATES[key]
            cur = table.get(key)
            best = cur
            for cand in cands:
                if cand == cur:
                    continue
                table[key] = cand
                tt = time_forward(m, x, t, ci)
                if tt < base * 0.996:
                    best, base = cand, tt
            if best is None:
                table.pop(key, None)
            else:
                table[key] = best
                plan._TUNED_NEW[key] = best
        final = time_forward(m, x, t, ci)
        print(f"channels {cfg['model_channels']} batch {n} size {hw}: {len(keys)} shapes, forward {start * 1e3:.1f} -> "
              f"{final * 1e3:.1f} us", flush=True)
    del m
    torch.cuda.empty_cache()


def main():
    which = sys.argv[1:] or ["decoder", "coarse", "base"]
    if "decoder" in which:
        run(O.DECODER_CFG, [(1, 256), (16, 256), (1, 512), (4, 512), (1, 64), (2, 256), (4, 256), (8, 256)])
    if "coarse" in which:
        run(COARSE_CFG, [(1, 64)], cond=lambda n: [torch.zeros(n, device="cuda") for _ in range(5)])
    if "base" in which:
        run(BASE_CFG, [(16, 64), (1, 64), (4, 64)], cond=lambda n: [torch.randn(n, 58, device="cuda")])
    table = {}
    try:
        table = json.load(open(plan.TUNED_PATH)).get("shapes", {})
    except Exception:
        pass
    table.update(plan._TUNED_NEW)
    json.dump({"device": torch.cuda.get_device_name(0), "how": "tools/tune_igemm.py: per-shape coordinate descent on the "
               "graph-replayed forward time", "shapes": dict(sorted(table.items()))}, open(plan.TUNED_PATH, "w"), indent=0)
    print("shapes in table:", len(table), "changed/measured in this run:", len(plan._TUNED_NEW))


if __name__ == "__main__":
    main()
