"""CPU: the `--impl reference` arm of bench.py (the reference's own CPU implementation, oracle/_ref when it compiles here,
else the oracle port) runs without a GPU and prints ONE JSON line with the contract's keys; the GPU arm must refuse to
produce a number without a GPU (no CPU fallback)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, cwd=ROOT, timeout=600)


import pytest


@pytest.mark.parametrize("cfg", [1, 2, 4])
def test_reference_arm_prints_one_contract_line(cfg):
    r = _run(["--impl", "reference", "--config", str(cfg), "--steps", "1", "--warmup", "1", "--ref-items-per-thread", "1", "--keyframes", "2000"])
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype",
              "data", "config", "impl", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "frames/s" and d["value"] > 0 and d["higher_is_better"] is True
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert f"configs[{cfg}]" in d["config"]["workload"]


def test_b200_arm_needs_a_gpu():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("GPU present: covered by the gpu-marked tests and the bench itself")
    r = _run(["--steps", "1", "--warmup", "1", "--pairs", "1", "--handles", "1", "--no-cpu-baseline"])
    assert r.returncode != 0                                       # loud failure, never a CPU-computed number
    assert not any(l.strip().startswith("{") and '"value"' in l for l in r.stdout.splitlines())


def test_reference_arm_under_torchrun_prints_on_rank_0_only():
    """The reference arm is launched like the GPU arm (torchrun, one process per GPU): rank 0 alone runs and prints
    the line, the other ranks exit 0 without output and without work."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29577", os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1",
           "--ref-items-per-thread", "1"]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip().startswith("{")]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 2 and d["value"] > 0
