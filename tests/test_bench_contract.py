"""bench.py's output contract: on the arm that runs without a GPU (`--impl reference`) exactly ONE
line on stdout, valid JSON, every key a caller reads; on the GPU arm, `--dump-outputs`."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_contract_line():
    proc = subprocess.run(
        [sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--arch", "tiny-gqa",
         "--exit-layer", "3", "--num-speculations", "4", "--steps", "1", "--warmup", "1",
         "--prompt-len", "12", "--cpu-max-steps", "8"],
        capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert proc.returncode == 0, proc.stderr[-2000:]
    lines = [l for l in proc.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, proc.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["unit"] == "tokens/s"
    for key in ("metric", "value", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "vs_baseline",
                "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in d, key
    assert d["value"] > 0 and d["e2e"]["value"] == d["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and "sample" in cb and cb["value"] == d["value"]
    assert "workload" in d["config"]


def test_non_zero_ranks_of_the_reference_arm_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    proc = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                          capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    assert proc.returncode == 0 and proc.stdout.strip() == ""


def test_usable_cpu_detection_is_sane():
    sys.path.insert(0, ROOT)
    import bench
    n = bench.usable_cpus()
    assert 1 <= n <= (os.cpu_count() or 1)
    assert 1 <= bench.cpu_threads() <= 32


@pytest.mark.gpu
def test_dump_outputs_writes_the_last_timed_generation(tmp_path):
    """`--dump-outputs DIR`: float64 .npy files of what the last timed generation returned to its
    caller, identical on a second run with the same arguments (seeded weights and prompts)."""
    import numpy as np
    args = [sys.executable, os.path.join(ROOT, "bench.py"), "--arch", "tiny-gqa", "--exit-layer", "3",
            "--num-speculations", "4", "--steps", "2", "--warmup", "1", "--prompt-len", "12",
            "--max-steps", "32", "--no-extra", "--no-cpu-baseline"]
    runs = []
    for i in range(2):
        out = tmp_path / f"run{i}"
        proc = subprocess.run(args + ["--dump-outputs", str(out)], capture_output=True, text=True,
                              timeout=600, cwd=ROOT)
        assert proc.returncode == 0, proc.stderr[-2000:]
        assert json.loads(proc.stdout.strip().splitlines()[-1])["steps"] == 2
        runs.append({n: np.load(out / f"{n}.npy") for n in ("tokens", "rounds", "acceptance_rate")})
    tokens, rounds = runs[0]["tokens"], runs[0]["rounds"]
    assert tokens.dtype == np.float64 and 1 <= tokens.size <= 32
    assert rounds.shape[1] == 3 and rounds[:, 2].sum() >= tokens.size      # emitted before EOS truncation
    for name in runs[0]:
        np.testing.assert_array_equal(runs[0][name], runs[1][name])
