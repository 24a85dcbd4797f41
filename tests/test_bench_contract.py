"""The CPU arm of bench.py (`--impl reference`) prints the contract's JSON line: checked here with a tiny sample
(ANCE_BENCH_TINY_CPU) so that the CPU suite stays fast; the GPU arm is exercised by the driver on an H100."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(extra_env):
    env = dict(os.environ, ANCE_BENCH_TINY_CPU="1", **extra_env)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "2",
                        "--warmup", "1"], capture_output=True, text=True, env=env, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    return [ln for ln in r.stdout.splitlines() if ln.startswith("{")]


def test_reference_arm_json_line():
    lines = _run({})
    assert len(lines) == 1
    d = json.loads(lines[0])
    base = json.load(open(os.path.join(ROOT, "BASELINE.json")))
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1
    assert d["higher_is_better"] is True and d["value"] > 0 and d["unit"] and d["metric"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert d["config"]["index_rows"] == 8841823 and d["config"]["topk"] == 200 and "workload" in d["config"]
    assert isinstance(base, dict)   # the metric string is free text; the config is what BASELINE.json's configs[1] names


def test_reference_arm_other_ranks_are_silent():
    assert _run({"RANK": "1", "WORLD_SIZE": "2"}) == []
