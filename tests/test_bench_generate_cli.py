"""tools/bench_generate.py times the GPU only: with no device visible it refuses instead of timing anything."""
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_refuses_without_a_gpu():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_generate.py"), "--workloads", "small"],
                       capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode != 0
    assert "no CUDA device" in r.stderr
    assert r.stdout.strip() == ""
