"""bench.py's reference arm runs on the CPU: check its one-line JSON contract here (the GPU arm needs an H100)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "groth16_withdraw_proofs_per_sec" and line["unit"] == "proofs/s"
    assert line["value"] > 0 and line["higher_is_better"] is True and line["steps"] == 1 and line["warmup"] == 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1 and line["cpu_baseline"]["value"] == line["value"]
    assert line["e2e"] == {"value": line["value"], "unit": "proofs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in line["config"] and line["gpu_launches"] == 0


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


@pytest.mark.gpu
def test_gpu_arm_dump_outputs(tmp_path):
    """--dump-outputs writes what the last timed step returned (proofs, public inputs) and the sharded MSM sums as float32
    .npy files of byte values; --steps sets the number of timed steps."""
    import numpy as np
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "2", "--warmup", "1",
                          "--batch", "4", "--no-cpu-baseline", "--no-parity", "--sharded-log-n", "12", "--dump-outputs", str(tmp_path)],
                         capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["steps"] == 2 and line["config"]["proofs_verify"] and line["sharded_msm"]["steps"] == 2
    shapes = {"proofs": (4, 256), "public_inputs": (4, 96), "sharded_msm_g1": (64,), "sharded_msm_g2": (128,)}
    for name, shape in shapes.items():
        a = np.load(tmp_path / f"{name}.npy")
        assert a.dtype == np.float32 and a.shape == shape, name
        assert np.all((a >= 0) & (a <= 255) & (a == np.round(a))) and a.any(), name


def test_launch_list_tool_reads_the_committed_ncu_csv(tmp_path):
    """tools/launch_list_summary.py turns an ncu launch list of the benchmark (the committed fixture under tests/golden/)
    into a per-kernel table: the dominant kernel of the bench command must come out on top."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = tmp_path / "ll.md"
    subprocess.run([sys.executable, os.path.join(root, "tools", "launch_list_summary.py"),
                    os.path.join(root, "tests", "golden", "ncu_launch_list.csv"), str(out), "t"], check=True)
    rows = [l for l in out.read_text().splitlines() if l.startswith("| `")]
    assert rows and rows[0].startswith("| `k_bucket_acc_sm1"), rows[:2]
