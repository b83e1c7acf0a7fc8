"""tools/bench_guided.py pieces that need no GPU: the GFLOP-per-step figure its roofline uses, computed from the conv /
attention shapes, reproduces the documented per-forward figures, and the tool declares the evaluation's workload."""
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

import bench  # noqa: E402
import bench_guided  # noqa: E402
from oracle import unet as ounet  # noqa: E402


def test_unet_gflop_reproduces_the_documented_forward_figures():
    # base 192x3 at 64^2: 193.65 GFLOP (SURVEY.md 8(d)); decoder at 256^2: 343.94 (BASELINE.md section 2).  Both
    # documented figures include the embedding linears, which unet_gflop leaves out (< 0.05 GFLOP).
    assert abs(bench_guided.unet_gflop(bench.BASE_CFG, 64) - bench.GFLOP_PER_LATENT_PHASE) < 0.05
    assert abs(bench_guided.unet_gflop(ounet.DECODER_CFG, 256) - bench.GFLOP_PER_STEP_256) < 0.05
    guide = bench_guided.unet_gflop(bench_guided.GUIDE_CFG, 64)
    assert 0.40 < guide / bench_guided.unet_gflop(bench.BASE_CFG, 64) < 0.50   # ~ (128/192)^2 of the main model


def test_guided_tool_declares_the_evaluation_workload():
    out = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_guided.py"), "--help"], capture_output=True,
                         text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "--tiles" in out.stdout and "--solve-steps" in out.stdout
    assert bench_guided.GUIDE_CFG == dict(bench.BASE_CFG, model_channels=128)
    assert (bench_guided.GUIDED_SCALE, bench_guided.GUIDED_STEPS, bench_guided.GUIDED_TILES) == (2.15, 32, 40)
