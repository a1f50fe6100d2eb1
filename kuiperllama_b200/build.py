"""Build libkllm_b200.so (the C-ABI product library) in-tree with nvcc for sm_90a.

Used by __graft_entry__.build(), tests and bench.py.  No JIT cache: the .so lands in
kuiperllama_b200/lib/, next to the sources it was built from.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
LIB = LIBDIR / "libkllm_b200.so"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _fingerprint() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*")) + [PKG.parent / "include" / "kllm_b200.h"]):
        if p.is_file():
            h.update(p.name.encode())
            h.update(p.read_bytes())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu under csrc/ into one shared library; no-op when up to date."""
    LIBDIR.mkdir(exist_ok=True)
    stamp = LIBDIR / ".stamp"
    fp = _fingerprint()
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == fp:
        return LIB
    objs = []
    objdir = LIBDIR / "obj"
    objdir.mkdir(exist_ok=True)
    common = [nvcc_path(), "-std=c++17", "-O3", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC",
              "-I", str(PKG.parent / "include")]
    if verbose:
        common += ["-Xptxas", "-v"]
    procs = []
    for src in _sources():
        obj = objdir / (src.stem + ".o")
        objs.append(obj)
        procs.append((src, subprocess.Popen(common + ["-c", str(src), "-o", str(obj)],
                                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        text = out.decode(errors="replace")
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"[kllm build] {src.name} FAILED\n{text}\n")
        elif verbose or text.strip():
            sys.stderr.write(f"[kllm build] {src.name}\n{text}\n")
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([nvcc_path(), *ARCH, "-shared", "-o", str(LIB), *map(str, objs)])
    stamp.write_text(fp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
