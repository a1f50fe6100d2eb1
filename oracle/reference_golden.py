"""Recorded outputs of the reference's own CUDA path, so that the bit-exactness checks against it run
on any machine, with or without oracle/_ref.

tests/golden/reference_cuda.json maps a check's key to what oracle/_ref (the reference's kernels and
model code compiled for sm_90a) produced on an H100 for the same seeded inputs: the SHA-256 of a float
output's bit pattern, or a list of token ids.  The checks compare our outputs against those records.

With KLLM_RECORD_REFERENCE=<json file> set (and oracle/_ref built), the checks instead run the
reference live, compare bit for bit as before, and add what the reference produced to that file --
which is how tests/golden/reference_cuda.json is made.

The stored records were made on an NVIDIA H100 80GB HBM3 (SXM, 700 W) with nvcc 12.9 (sm_90a) and torch 2.11
(its CUDA generator draws the seeded inputs), by `KLLM_RECORD_REFERENCE=<file> python -m pytest -m gpu tests`
and `smoke()` on that GPU; the CPU-orchestration entries by `KLLM_RECORD_REFERENCE=<file> python -m pytest
tests/test_oracle_golden.py`.  A GPU run is needed to check them, since the inputs come from the CUDA RNG.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
from __future__ import annotations

import hashlib
import json
import os
from pathlib import Path

import numpy as np

GOLDEN_FILE = Path(__file__).resolve().parent.parent / "tests" / "golden" / "reference_cuda.json"


def _f32(a):
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.ascontiguousarray(a, dtype=np.float32)


def digest(a) -> str:
    """SHA-256 of the float32 bit pattern (distinguishes -0.0 and NaN payloads), 32 hex digits."""
    return hashlib.sha256(_f32(a).view(np.uint32).tobytes()).hexdigest()[:32]


class Reference:
    """`live`: the reference library is loaded (`.L`) and every check records what it produced."""

    def __init__(self, flavour: str = "llama2"):
        self.record_to = os.environ.get("KLLM_RECORD_REFERENCE")
        self.live = bool(self.record_to)
        if self.live:
            from oracle.binding import RefCuda
            self.L = RefCuda(flavour).L
        self.table = json.loads(GOLDEN_FILE.read_text()) if GOLDEN_FILE.exists() else {}

    def _record(self, key, value):
        path = Path(self.record_to)
        table = json.loads(path.read_text()) if path.exists() else {}
        table[key] = value
        path.write_text(json.dumps(table, indent=0, sort_keys=True) + "\n")

    def _want(self, key):
        if key not in self.table:
            raise AssertionError(f"no recorded reference output for {key!r} in {GOLDEN_FILE.name}")
        return self.table[key]

    def bits(self, key, ours, theirs=None, what=""):
        """`ours` must equal the reference's output bit for bit (`theirs` when live)."""
        a = _f32(ours)
        if self.live:
            b = _f32(theirs)
            self._record(key, digest(b))
            bad = np.nonzero(a.view(np.uint32).ravel() != b.view(np.uint32).ravel())[0]
            assert a.shape == b.shape and bad.size == 0, \
                f"{what or key}: {bad.size}/{a.size} elements differ bitwise from the reference CUDA path"
        else:
            assert digest(a) == self._want(key), \
                f"{what or key}: differs bitwise from the reference CUDA path's recorded output"

    def ids(self, key, ours, theirs=None, what=""):
        """Token ids (or any list of ints) equal to the reference's."""
        ours = [int(v) for v in ours]
        if self.live:
            theirs = [int(v) for v in theirs]
            self._record(key, theirs)
        else:
            theirs = self._want(key)
        assert ours == theirs, f"{what or key}: ids differ from the reference CUDA path"
