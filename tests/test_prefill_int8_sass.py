"""The int8 prefill GEMM and its measurement tool without a GPU: what the compiler made of the kernel, and a
timing tool that refuses to run rather than time anything off the device."""
import re
import subprocess
import sys

import pytest

from conftest import ROOT


def test_int8_weight_prefill_gemms_run_on_the_tensor_cores_without_local_memory(kllm_lib):
    """Every instantiation of gemm_tf32_kernel for int8 weights (kllm_gemm_w8_tf32) is fed by TMA (UTMALDG) and
    multiplies with wgmma (HGMMA), with no stack and no local-memory access: its 128 accumulators per thread at
    BN = 256 live in registers."""
    from kuiperllama_b200 import build as kbuild
    lib = str(kbuild.LIB)
    res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = {m.group(1): int(m.group(2))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", res)}
    w8 = sorted(n for n in usage if "gemm_tf32_kernel" in n and re.search(r"ILi\d+ELNS_12WeightFormatE1E", n))
    assert len(w8) == 4, sorted(n for n in usage if "gemm_tf32_kernel" in n)  # BN = 32, 64, 128, 256
    for name in w8:
        assert usage[name] == 0, f"{name}: {usage[name]} bytes of stack"
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", name, lib], capture_output=True, text=True,
                              check=True).stdout
        assert "HGMMA" in sass and "UTMALDG" in sass, name
        assert not re.search(r"\b(?:LDL|STL)\b", sass), f"{name}: local-memory instructions"


def test_prefill_timing_tool_needs_cuda():
    """tools/bench_prefill.py times GPU paths only: without a device it fails and prints nothing."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, str(ROOT / "tools" / "bench_prefill.py"), "--workload", "small",
                        "--tokens", "8"], capture_output=True, text=True, timeout=300, cwd=str(ROOT))
    assert r.returncode != 0 and r.stdout.strip() == ""
