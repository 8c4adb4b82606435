"""bench.py contract checks that need no GPU: the reference arm (`--impl reference`, the oracle port timed on host
cores) prints ONE JSON line with the result keys; per-GPU batch of the configs BASELINE.json quotes as 8-GPU
global batches."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--config", "cfg1", "--steps", "1",
                        "--warmup", "1", "--cpu-sample", "2"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["higher_is_better"] is True and d["unit"] == "pairs/s"
    for k in ("metric", "value", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "vs_baseline", "dtype", "data", "config",
              "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["value"] > 0 and d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]


def test_per_gpu_batch_of_the_eight_gpu_configs():
    sys.path.insert(0, ROOT)
    import bench
    assert bench.build_cfg("cfg2")["B"] == 256          # quoted on 1 GPU
    assert bench.build_cfg("cfg3")["B"] == 512 // 8     # global batch over 8 data-parallel ranks
    assert bench.build_cfg("cfg4")["B"] == 256 // 8
    assert bench.build_cfg("cfg5")["B"] == 1024 // 8
    assert bench.build_cfg("cfg5", 16)["B"] == 16
    assert "configs[4]" in bench.workload_name(bench.build_cfg("cfg5"))
