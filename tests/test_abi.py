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


def test_megakernel_keeps_its_state_out_of_local_memory(kllm_lib):
    """The persistent kernel's ring takes the whole unified L1, so a local-memory access is a round trip to L2
    (DESIGN.md 5.2, "No local memory").  Gate: the default instantiations -- 8 fp32 and 8 int8 consumer warps --
    carry no parameter copy on the stack (it was 456 bytes before the parameters became __grid_constant__) and
    only a handful of local loads / stores (per-token spills and the cold trap-message path), none of them in
    the row loops' register budget class; nvcc / ptxas regressions of that kind show up here, on the CPU."""
    import re
    import subprocess
    from kuiperllama_b200 import build as kbuild
    lib = str(kbuild.LIB)
    res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", res):
        usage[m.group(1)] = (int(m.group(2)), int(m.group(3)))
    defaults = {"_ZN4kllm4mega17decode_megakernelILi8ELb0ELb0EEEvNS0_6ParamsE": 168,
                "_ZN4kllm4mega17decode_megakernelILi8ELb1ELb0EEEvNS0_6ParamsE": 168}
    # one consumer-warp count: {fp32, int8} x {plain, profiling}
    assert sorted(k for k in usage if "decode_megakernel" in k) == sorted(
        f"_ZN4kllm4mega17decode_megakernelILi8ELb{int8}ELb{prof}EEEvNS0_6ParamsE" for int8 in (0, 1) for prof in (0, 1))
    for name, reg_cap in defaults.items():
        assert name in usage, sorted(k for k in usage if "megakernel" in k)
        regs, stack = usage[name]
        assert regs <= reg_cap, (name, regs)
        assert stack <= 64, f"{name}: {stack} bytes of stack (a parameter copy or a local array is back)"
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", name, lib], capture_output=True, text=True, check=True).stdout
        local = len(re.findall(r"\b(?:LDL|STL)\b", sass))
        assert local <= 32, f"{name}: {local} local-memory instructions"
        assert "UBLKCP" in sass and "SYNCS" in sass  # TMA bulk copies + mbarriers are what feeds the ring
