"""The drop-in boundary without a GPU: the C-ABI library builds for sm_90a, loads, exports
exactly what include/kllm_b200.h declares, does not depend on the oracle, and the Python
loader fails loudly when the library is absent."""
import re
import subprocess

import pytest

from kuiperllama_b200 import HEADER_PATH, LIB_PATH, KllmError, _SIGNATURES, load_library


def header_functions():
    text = HEADER_PATH.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = re.findall(r"\b(kllm_[a-z0-9_]+)\s*\(", text)
    # drop the struct-member callback and type names
    return sorted(set(n for n in names if n not in ("kllm_decoder",)))


def test_every_declared_symbol_is_exported(kllm_lib):
    declared = header_functions()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(kllm_lib, name), f"{name} declared in kllm_b200.h but not exported"
        assert name in _SIGNATURES, f"{name} has no ctypes prototype"
    assert sorted(_SIGNATURES) == declared


def test_library_is_sm90a_and_oracle_free(kllm_lib):
    sass = subprocess.run(["cuobjdump", "-lelf", str(LIB_PATH)], capture_output=True, text=True).stdout
    assert "sm_90a" in sass, sass
    syms = subprocess.run(["nm", "-D", str(LIB_PATH)], capture_output=True, text=True).stdout
    assert "ko_" not in syms and "kref_" not in syms, "product library must not contain oracle code"
    deps = subprocess.run(["ldd", str(LIB_PATH)], capture_output=True, text=True).stdout
    assert "oracle" not in deps and "kuiper_ref" not in deps


def test_product_sources_never_touch_the_oracle():
    from pathlib import Path
    pkg = Path(LIB_PATH).parent.parent
    for p in list(pkg.rglob("*.py")) + list(pkg.rglob("*.cu")) + list(pkg.rglob("*.cuh")) + \
            list(pkg.rglob("*.h")) + list(pkg.rglob("*.cpp")) + list(pkg.rglob("CMakeLists.txt")):
        text = p.read_text(errors="replace")
        assert "kuiper_oracle" not in text and "oracle.binding" not in text and \
            "liboracle" not in text, f"{p} references the oracle"


def test_library_reads_only_the_documented_environment(kllm_lib):
    """Every KLLM_ environment variable the library reads: the engine, the numerics mode, and the ring-stage
    size and attention split that the decode-model tests use to reach ring geometries.  An option that nothing
    sets is a code path that nothing tests, so a new name has to be added here on purpose."""
    data = LIB_PATH.read_bytes()
    names = {m.decode() for m in re.findall(rb"(?<![A-Za-z0-9_])KLLM_[A-Z0-9_]+(?=\x00)", data)}
    assert names == {"KLLM_ENGINE", "KLLM_MODE", "KLLM_STAGE_BYTES", "KLLM_ATTN_SPLIT"}


def test_missing_library_fails_loudly(tmp_path):
    with pytest.raises(KllmError):
        load_library(tmp_path / "libkllm_b200.so")


def test_version_and_error_strings(kllm_lib):
    assert b"sm_90a" in kllm_lib.kllm_version()
    assert kllm_lib.kllm_error_string(-1) == b"invalid argument"


def test_argument_validation_without_device(kllm_lib):
    # pure host-side checks: must return KLLM_E_INVALID before touching CUDA
    assert kllm_lib.kllm_gemv_f32(None, None, None, 4, 4, None) == -1
    assert kllm_lib.kllm_rmsnorm_f32(None, None, None, 0, 1e-5, None) == -1
    assert kllm_lib.kllm_decoder_create(None, None, None) == -1


def test_every_megakernel_instantiation_keeps_its_state_out_of_local_memory(kllm_lib):
    """The persistent kernel's ring takes the whole unified L1, so a local-memory access is a round trip to L2
    (DESIGN.md 5.2, "No local memory").  The library holds exactly the decode_megakernel<F, KV, LP, PROF>
    instantiations of tests/megakernel_table.py -- {fp32, int8, bf16} weights x {fp32, bf16, fp8} caches x {plain,
    log-probabilities}, plus the profiling kernels of fp32 and int8 weights over the fp32 cache -- and every one of
    them carries no parameter copy on the stack (it was 456 bytes before the parameters became __grid_constant__) and
    only a handful of local loads / stores (per-token spills and the cold trap-message path), is fed by TMA bulk copies
    on mbarriers, and with the fp8 cache widens and encodes e4m3 in hardware.  The plain fp32 and int8 kernels over the
    fp32 cache keep the row loops' register budget.  nvcc / ptxas regressions of that kind show up here, on the CPU."""
    from megakernel_table import TABLE, symbol
    from kuiperllama_b200 import build as kbuild
    lib = str(kbuild.LIB)
    res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", res)}
    name = {t: symbol(*t) for t in TABLE}
    assert len(name) == 20
    assert sorted(k for k in usage if "megakernel" in k) == sorted(name.values())
    for (f, kv, lp, prof), n in name.items():
        regs, stack = usage[n]
        assert stack <= 64, f"{n}: {stack} bytes of stack (a parameter copy or a local array is back)"
        if f != "bf16" and kv == "fp32" and not lp and not prof:
            assert regs <= 168, (n, regs)
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", n, lib], capture_output=True, text=True, check=True).stdout
        local = len(re.findall(r"\b(?:LDL|STL)\b", sass))
        assert local <= 32, f"{n}: {local} local-memory instructions"
        assert "UBLKCP" in sass and "SYNCS" in sass, n  # TMA bulk copies + mbarriers are what feeds the ring
        if kv == "fp8":
            assert "F2FP.F16.E4M3.UNPACK_B" in sass and "SATFINITE.E4M3" in sass, n  # hardware e4m3 conversions
