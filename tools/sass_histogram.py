#!/usr/bin/env python
"""Instruction histogram of the kernels in libkllm_b200.so (cuobjdump -sass), per kernel: total
instructions and the mnemonics that prove which hardware paths are used (TMA bulk copies, wgmma,
mbarriers, dp4a, ...).

    python tools/sass_histogram.py > profiles/r02_sass_histogram.txt
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "kuiperllama_b200" / "lib" / "libkllm_b200.so"
KEY = ["UBLKCP", "UBLKPF", "UTMALDG", "UTMASTG", "UTCHMMA", "UTCQMMA", "UTCIMMA", "LDTM", "STTM", "UTCBAR", "UTCATOMSWS", "IMMA",
       "SYNCS", "IDP", "FFMA", "FADD", "FMUL", "PRMT", "I2F", "LDS", "STS", "LDG", "STG", "LD", "ST", "SHFL", "MUFU",
       "BAR", "HMMA", "NANOSLEEP", "CCTL", "ATOM", "RED", "MEMBAR", "LDL", "STL"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = kernels.setdefault(m.group(1), collections.Counter())
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and cur is not None:
            cur[m.group(1)] += 1
    demangle = subprocess.run(["c++filt"], input="\n".join(kernels), capture_output=True, text=True).stdout.splitlines()
    print(f"# {LIB.name}: SASS instruction histogram per kernel (sm_90a, cuobjdump -sass); mnemonic families summed over suffixes")
    for (mangled, cnt), name in zip(kernels.items(), demangle):
        fam = collections.Counter()
        for op, n in cnt.items():
            fam[op.split(".")[0]] += n
        total = sum(cnt.values())
        shown = [f"{k} {fam[k]}" for k in KEY if fam.get(k)]
        dp4a = sum(n for op, n in cnt.items() if op.startswith("IDP.4A"))
        print(f"\n{name}\n  {total} instructions; " + ", ".join(shown) + (f"; IDP.4A {dp4a}" if dp4a else ""))
    return 0


if __name__ == "__main__":
    sys.exit(main())
