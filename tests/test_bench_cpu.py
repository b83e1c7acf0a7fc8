"""bench.py contract pieces that need no GPU: the reference arm (`--impl reference`, the CPU oracle port timed on the host
cores) prints ONE JSON line with the keys the driver reads, on the same metric / unit / config as the GPU arm."""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_reference_arm_prints_the_contract_line():
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "tile-steps/s" and d["higher_is_better"] is True
    assert d["metric"].startswith("denoising steps/sec") and d["n_gpus"] == 1 and d["value"] > 0
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["sample"]
    assert "workload" in d["config"]


def test_gpu_arms_are_declared():
    src = (ROOT / "bench.py").read_text()
    for flag in ("--gpus", "--steps", "--warmup", "--impl", "--tiles", "--size", "--workload"):
        assert flag in src
    for w in ("tiles", "canvas", "export", "latent", "world"):
        assert f'"{w}"' in src


def test_committed_headline_line_carries_every_contract_key():
    """The bench line kept under profiles/ (an H100 run of the default workload) has every key of the result line."""
    d = json.loads((ROOT / "profiles" / "bench_tiles1.json").read_text())
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"):
        assert k in d, k
    assert d["n_gpus"] == 1 and d["unit"] == "tile-steps/s" and d["dtype"] == "bf16" and d["vs_baseline"] is None
    r = d["roofline"]
    assert r["bound"] == "tensor" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and r["traffic"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] < d["value"] * 1.01
    assert d["cpu_baseline"]["kind"] == "port" and d["gpu_launches"] > 0
    assert not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert "workload" in d["config"] and "l2" in d["config"]
