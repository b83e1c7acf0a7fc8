"""Per-launch device times of one forward (eager, CUDA events around each launch) with shapes and TFLOP/s."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from oracle import unet as O
from terrain_diffusion_b200.models import EDMUnet2D


def main():
    size = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    cfg = O.DECODER_CFG
    m = EDMUnet2D(**cfg).eval()
    m.load_state_dict(O.procedural_state_dict(cfg, seed=0))
    m = m.cuda()
    x = torch.randn(n, 5, size, size, device="cuda")
    t = torch.full((n,), 1.2, device="cuda")
    m(x, t, [])
    prog, bufs = m._plans[("fwd", n, size, size, False)]
    best = None
    for _ in range(5):
        ms, kinds = prog.profile()
        if best is None:
            best = ms
        else:
            best = [min(a, b) for a, b in zip(best, ms)]
    names = {1: "igemm", 2: "conv_out", 3: "embed", 4: "attn", 5: "im2col"}
    tot = sum(best)
    print(f"forward {size}x{size} N={n}: sum of per-launch times {tot*1e3:.1f} us over {len(best)} launches")
    agg = {}
    for i, (t_, k) in enumerate(zip(best, kinds)):
        agg[names[k]] = agg.get(names[k], 0.0) + t_
    for k, v in agg.items():
        print(f"  {k:9s} {v*1e3:9.1f} us  {v/tot:6.1%}")
    print("per-launch us:", " ".join(f"{t_*1e3:.1f}" for t_ in best))


if __name__ == "__main__":
    main()
