"""CPU: the prompt-lookup drafting rule and the round structure of speculative decoding (speculative.py, stated in
include/kllm_b200.h), the new C-ABI declarations and symbols, and the verify kernels' local-memory gate."""
import re
import subprocess
from pathlib import Path

import pytest

from kuiperllama_b200.speculative import lookup_draft, simulate_rounds

HEADER = Path(__file__).resolve().parents[1] / "include" / "kllm_b200.h"


def test_largest_n_first():
    # the 2-gram (4, 5) matches at s = 1 -> draft [6, 7]; the 1-gram (5) alone would match later at s = 5 -> [9]
    c = [3, 4, 5, 6, 7, 5, 9, 4, 5]
    assert lookup_draft(c, 2, 4) == [6, 7, 5, 9]
    assert lookup_draft(c, 1, 4) == [9, 4, 5]


def test_latest_match_wins():
    c = [1, 2, 10, 1, 2, 20, 1, 2]
    assert lookup_draft(c, 2, 3) == [20, 1, 2]
    assert lookup_draft(c, 2, 1) == [20]


def test_holes_in_the_history():
    # a suffix with -1 is skipped; a draft stops at the first -1
    assert lookup_draft([5, 6, -1, 5, 6], 2, 4) == []  # the match at 0 runs into the hole at once
    assert lookup_draft([5, 6, 7, -1, 5, 6], 2, 4) == [7]
    assert lookup_draft([1, 2, -1, 2], 2, 4) == []  # suffix (-1, 2) skipped; 1-gram 2 at s = 1 drafts -1: empty
    assert lookup_draft([-1, 3, 4, 3], 3, 4) == [4, 3]  # n = 3 and 2 match only across the -1; n = 1 matches at 1


def test_caps_and_empty_drafts():
    c = [1, 2, 3, 4, 1, 2]
    assert lookup_draft(c, 2, 0) == []
    assert lookup_draft(c, 2, 2) == [3, 4]
    assert lookup_draft(c, 2, 7) == [3, 4, 1, 2]  # a draft ends at the context's end
    assert lookup_draft([9], 3, 4) == []  # too short for any match
    assert lookup_draft([1, 2, 3], 3, 4) == []  # no repeat
    assert lookup_draft([4, 4], 8, 4) == [4]  # the match may overlap the suffix's own start


def test_simulate_rounds_on_constructed_streams():
    kw = dict(draft_len=4, ngram_max=2, max_steps=100, seq_len=1000)
    # context [1, 2, 3, 1, 2]: round 1 drafts [3, 1, 2] (cap: only 3 ids follow), all accepted plus one more id
    assert simulate_rounds([1, 2, 3, 1, 2], [3, 1, 2, 3], **kw) == {"rounds": 1, "drafted": 3, "accepted": 3}
    # the first draft id is wrong: one id from the round
    r = simulate_rounds([1, 2, 3, 1, 2], [8], **kw)
    assert r == {"rounds": 1, "drafted": 3, "accepted": 0}
    # no draft at all: plain steps, one id each
    assert simulate_rounds([7], [8, 9], **kw) == {"rounds": 2, "drafted": 0, "accepted": 0}
    # a stop id ends the acceptance at its position
    r = simulate_rounds([1, 2, 3, 1, 2], [3, 1], stop_ids=[1], **kw)
    assert r == {"rounds": 1, "drafted": 3, "accepted": 1}
    # max_steps caps the draft: max_steps - produced - 1
    r = simulate_rounds([1, 2, 3, 1, 2], [3, 1], **dict(kw, max_steps=2))
    assert r == {"rounds": 1, "drafted": 1, "accepted": 1}
    # seq_len caps it too: seq_len - p - 1 with p = 4
    r = simulate_rounds([1, 2, 3, 1, 2], [3, 1, 2], **dict(kw, seq_len=7))
    assert r == {"rounds": 1, "drafted": 2, "accepted": 2}


def test_header_declares_the_entries(kllm_lib):
    text = HEADER.read_text()
    assert "#define KLLM_MAX_VERIFY_TOKENS 8" in text
    for name in ("kllm_decoder_verify", "kllm_decoder_generate_speculative"):
        assert re.search(rf"\bint {name}\(", text), name
        assert getattr(kllm_lib, name) is not None
    assert re.search(r"typedef struct \{\s*int32_t rounds;\s*int32_t drafted;\s*int32_t accepted;\s*\} kllm_spec_stats;",
                     text)


def test_verify_kernels_keep_out_of_local_memory(kllm_lib):
    """The verify chain's kernels stay out of local memory: none at all for the embedding, accept and attention
    kernels; the draw block carries the sampling helpers it shares with argmax_advance_kernel (sampling.cuh
    draw_and_record) and a per-position copy of the step-0 settings; the multi-vector GEMV may keep an 8-byte frame,
    with a few accesses to it."""
    from kuiperllama_b200 import build as kbuild
    lib = str(kbuild.LIB)
    res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", res)}
    names = [k for k in usage if re.search(r"gemv_multi_kernel|verify_\w+_kernel|mha_decode_kernelILb1", k)]
    assert len(names) == 6 + 3 + 1, names
    for name in names:
        regs, stack = usage[name]
        gemv = "gemv_multi" in name
        assert stack <= (64 if "verify_draw" in name else 8 if gemv else 0), (name, stack)
        sass = subprocess.run(["cuobjdump", "-sass", "-fun", name, lib], capture_output=True, text=True,
                              check=True).stdout
        assert len(re.findall(r"\b(?:LDL|STL)\b", sass)) <= (48 if "verify_draw" in name else 16 if gemv else 0), name
