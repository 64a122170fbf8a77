"""`bench.py --impl reference` (the CPU arm beside the GPU arm) prints one contract-shaped JSON line.
Runs the C/OpenMP oracle on a CI-sized preset; nothing here touches a GPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    # OMP_NUM_THREADS=1 is what torchrun exports to its workers: the arm must size its own team (VERDICT r1)
    env = dict(os.environ, OMP_NUM_THREADS="1", B200RWKV_CPU_THREADS="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1",
                          "--preset", "small6", "--batch", "4"],
                         capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "tokens/s" and line["higher_is_better"] is True
    assert line["value"] > 0 and line["steps"] == 2 and line["n_gpus"] == 1
    cb = line["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] == 2 and cb["value"] == line["value"]
    assert "small6" in line["metric"] and "batch=4" in line["metric"]
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
    assert "workload" in line["config"]


def test_reference_arm_other_ranks_exit_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1", B200RWKV_BENCH_PRESET="tiny6")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1"],
                         capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_host_threads_is_positive():
    sys.path.insert(0, ROOT)
    import bench
    assert bench.host_threads() >= 1
