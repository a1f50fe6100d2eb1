"""Beam search over a batch of decoders (kllm_batch_beam_search, DESIGN.md 5.16), stated once in Python.

The rule is transformers' GenerationMixin._beam_search (5.5.0) for one sequence and B beams, with no logits
processors, over the log-probabilities of rule L1-L3 (sampling.logprobs).  The C++ host loop in decoder.cu
(run_batch_beam) applies the same steps in the same order, so both give the same bits.  t is the number of ids
generated so far, this pass's included; n_eos the number of eos ids.

1. Running beams.  Beam b has a running sum S_b (fp32).  Pass 0 has one beam, S = 0: transformers' start of
   [0, -1e9, ...] is the same when vocab >= K = max(2, 1 + n_eos) * B, which the entry requires.
2. Candidates.  Each running beam offers its first B + n_eos ids of the logprob rule's top-N order (logit
   descending, lowest id on ties) with their L3 values lp, scored s = fp32(S_b + lp).  All candidates are ordered by s
   descending, then beam index ascending, then the beam's own order.  That is enough to reproduce transformers' top-K:
   at most B of the global top-B ranks come from one beam, and a beam's best B non-eos ids lie within its first
   B + n_eos.
3. Finished hypotheses.  Each of the first B ranks that is an eos id -- every one of them when t = max_new_tokens --
   is offered as a finished hypothesis (its ids end with that id) with score h = fp32(s / fp32(t ** alpha)): torch
   divides a float32 tensor by a Python float by rounding the float (here the double t ** alpha, C's pow) to float32
   and dividing in float32, which tests/test_beam_rule.py checks.  Offers merge into B slots that start empty, keeping
   the B best by h; on equal h a slot already held stays ahead of an offer, and offers keep their rank order.  Nothing
   is offered once every slot is full and early_stopping is True, nor once the early-stop heuristic is satisfied
   (_update_finished_beams' two -1e9 gates).
4. Next beams.  The first B candidates that are not eos ids, in the order of 2, each with S = s.
5. Stop.  After each pass the heuristic is updated (_check_early_stop_heuristic): it stays unsatisfied while some slot
   is empty or fp32(S_0 / fp32(L ** alpha)) > the worst slot's h, with S_0 the best next beam's sum, L =
   max_new_tokens for early_stopping "never" with alpha > 0, else t; once satisfied it stays so.  The search stops when
   the heuristic is satisfied, when every slot is full and early_stopping is True
   (_beam_search_has_unfinished_sequences), or after the pass at t = max_new_tokens.
6. Result.  The filled slots in order of h descending (every slot is filled by the time the search stops); the first
   n_return are returned with their ids, h and S.

The members' cache forks (DESIGN.md 5.16) follow from the beams: after pass 0 member 0's rows [0, start_pos] go to
members 1 .. B - 1 (B - 1 forks of start_pos + 1 rows, made even when the search stops there), and after a later pass
p that another pass follows, a beam whose parent already gave its member to an earlier child takes a dropped beam's
member and receives the generated rows [start_pos + 1, start_pos + p]: B - (distinct parents) forks of p rows.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

EARLY_STOPPING = {False: 0, True: 1, "never": 2}  # KLLM_BEAM_EARLY_HEURISTIC / _ALL_DONE / _NEVER


@dataclass(frozen=True)
class Beam:
    """A running beam: the ids generated so far, the index of its beam in the previous pass (-1 at pass 0) and S."""
    ids: tuple
    parent: int
    sum: np.float32


def length_divisor(length: int, alpha: float) -> np.float32:
    """fp32(length ** alpha): Python's power of the int and the float (C's pow), rounded once to float32."""
    return np.float32(math.pow(float(length), float(alpha)))


def early_stopping_code(early_stopping) -> int:
    """transformers' early_stopping value (False, True or "never") as the C entry's code."""
    for k, v in EARLY_STOPPING.items():
        if early_stopping is k or (isinstance(k, str) and early_stopping == k):
            return v
    raise ValueError(f"early_stopping={early_stopping!r}: False, True or 'never'")


def beam_search(candidates, n_beams: int, max_new_tokens: int, eos_ids=(), length_penalty: float = 1.0,
                early_stopping=False, n_return: int = 1, start_pos: int = 0):
    """The rule above.  `candidates(beams)` receives the running beams (a list of Beam) and returns, for each, its
    (ids, lp) in the logprob rule's top-N order, at least n_beams + len(eos_ids) of them.  Returns (hypotheses,
    stats): the first n_return slots as dicts {"ids", "score" (h), "sum" (S)}, and {"passes", "forks", "fork_rows"}
    of the members' cache forks for a search whose prompt ends at start_pos."""
    B = int(n_beams)
    eos = [int(e) for e in eos_ids]
    eos_set = set(eos)
    top = B + len(eos)
    mode = early_stopping_code(early_stopping)
    alpha = float(length_penalty)
    beams = [Beam((), -1, np.float32(0.0))]
    slots = []  # (h, S, ids), h descending
    unsatisfied = True
    stats = {"passes": 0, "forks": 0, "fork_rows": 0}
    for t in range(1, int(max_new_tokens) + 1):
        per_beam = candidates(beams)
        stats["passes"] += 1
        cands = []  # (s, beam, k, id): the sort key is (-s, beam, k)
        for b, (ids, lps) in enumerate(per_beam):
            ids, lps = list(ids)[:top], np.asarray(lps, np.float32)[:top]
            for k in range(top):
                cands.append((np.float32(beams[b].sum + lps[k]), b, k, int(ids[k])))
        cands.sort(key=lambda c: (-c[0], c[1], c[2]))
        last = t == max_new_tokens
        full = len(slots) == B
        if unsatisfied and not (full and mode == 1):
            div = length_divisor(t, alpha)
            offers = [(np.float32(s / div), s, beams[b].ids + (i,)) for s, b, _, i in cands[:B]
                      if last or i in eos_set]
            merged = slots + offers
            merged.sort(key=lambda h: -h[0])  # stable: held slots first, then offers in rank order
            slots = merged[:B]
        nxt = [Beam(beams[b].ids + (i,), b, s) for s, b, _, i in cands if i not in eos_set][:B]
        full = len(slots) == B
        if unsatisfied:
            L = max_new_tokens if (mode == 2 and alpha > 0.0) else t
            best = np.float32(nxt[0].sum / length_divisor(L, alpha))
            unsatisfied = not full or bool(best > min(h for h, _, _ in slots))
        stop = last or not unsatisfied or (full and mode == 1)
        if t == 1 and B > 1:
            stats["forks"] += B - 1
            stats["fork_rows"] += (B - 1) * (start_pos + 1)
        elif not stop:
            forks = B - len({nb.parent for nb in nxt})
            stats["forks"] += forks
            stats["fork_rows"] += forks * (t - 1)
        if stop:
            break
        beams = nxt
    hyps = [{"ids": list(ids), "score": h, "sum": S} for h, S, ids in slots[:n_return]]
    return hyps, stats
