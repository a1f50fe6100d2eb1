"""Prompt-lookup drafting and the round structure of kllm_decoder_generate_speculative, in Python.

The decoder drafts on the host from its history and checks each draft with one verify pass (DESIGN.md 5.13).  This
module states the same rule, so that tests and tools/bench_speculative.py can predict a run's rounds, drafted and
accepted counts exactly from the ids it produced: given those ids, every round's draft and acceptance is determined.
"""
from __future__ import annotations

# draft ids per verify pass unless the caller chooses: the cheapest pass that can accept a draft, since a pass costs
# more with every position whether or not its drafts are accepted (DESIGN.md 5.13)
DEFAULT_DRAFT_LEN = 2


def lookup_draft(context, ngram_max: int, draft_len_cap: int) -> list[int]:
    """The draft for the position after `context` (the history up to the next position, then the id fed there).

    For n = ngram_max down to 1: skip n when the suffix context[L-n:] has fewer than n ids or contains -1; else find
    the largest s with s + n <= L - 1 and context[s:s+n] equal to the suffix.  The draft is context[s+n:], cut at the
    first -1 and after draft_len_cap ids.  The first n whose draft is not empty wins; [] means a plain step."""
    c = [int(t) for t in context]
    L = len(c)
    if draft_len_cap <= 0:
        return []
    for n in range(ngram_max, 0, -1):
        if L < n:
            continue
        suffix = c[L - n:]
        if any(t < 0 for t in suffix):
            continue
        for s in range(L - 1 - n, -1, -1):
            if c[s:s + n] != suffix:
                continue
            draft = []
            for t in c[s + n:]:
                if t < 0 or len(draft) == draft_len_cap:
                    break
                draft.append(t)
            if draft:
                return draft
            break  # the largest match decides this n
    return []


def simulate_rounds(context, ids, *, draft_len: int, ngram_max: int, max_steps: int, seq_len: int,
                    stop_ids=()) -> dict:
    """The rounds of kllm_decoder_generate_speculative that produced `ids`, from `context` (the history before the
    start position, then the first id).  Returns {"rounds", "drafted", "accepted"}."""
    c = [int(t) for t in context]
    ids = [int(t) for t in ids]
    stops = {int(t) for t in stop_ids}
    start = len(c) - 1
    produced = rounds = drafted = accepted = 0
    while produced < len(ids):
        p = start + produced
        m = min(draft_len, max_steps - produced - 1, seq_len - p - 1)
        draft = lookup_draft(c, ngram_max, m)
        a = 0
        while a < len(draft) and produced + a < len(ids) and draft[a] == ids[produced + a] \
                and ids[produced + a] not in stops:
            a += 1
        rounds += 1
        drafted += len(draft)
        accepted += a
        c += ids[produced:produced + a + 1]
        produced += a + 1
    return {"rounds": rounds, "drafted": drafted, "accepted": accepted}
