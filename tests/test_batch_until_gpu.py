"""-m gpu: kllm_batch_generate_until -- each member of a batch stops on its own stop ids or its own max_steps, with
its ids streamed while the loop runs -- against twin decoders over the same weights that run their own
generate_until, bit for bit: ids, the callbacks' concatenation, logits, history, log-probability record (with the
persistent engine's last-bits exception on the log-probabilities) and the WHOLE KV cache, so that nothing past a
member's end was written.  Stop ids come from a third decoder per member, a probe that runs the same continuation
with generate, so the twins' and members' caches hold nothing past their ends."""
import ctypes
from dataclasses import replace

import numpy as np
import pytest

from decode_model_util import GEOMETRIES
from gpu_util import assert_bit_equal
from kuiperllama_b200 import (BATCH_TOKEN_CALLBACK, MAX_BATCH, MAX_STOP_IDS, SHAPES, Batch, BatchStats, Decoder,
                              KllmError, synth_weights)
from kuiperllama_b200.decoder import bf16_weights
from test_batch_gpu import GRAPH_ONLY, SETTINGS, assert_unchanged, snapshot

pytestmark = pytest.mark.gpu

E_INVALID = -1


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def trio(shape, engine, n, weight_format="fp32", seed=2024, top_n=5):
    """n members, n twins and n probes over one weight set, each with logprobs top_n."""
    w = synth_weights(shape, "cuda", seed)
    if weight_format == "bf16":
        w = bf16_weights(w)
    try:
        ds = [Decoder(shape, w, weight_format=weight_format) for _ in range(3 * n)]
    except KllmError:
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    if ds[0].engine != engine:
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    for d in ds:
        d.set_logprobs(top_n)
    return ds[:n], ds[n:2 * n], ds[2 * n:]


def feed(groups, lengths, vocab):
    """Member b of every group fed a prompt of lengths[b] ids; returns the ids each continues with."""
    firsts = []
    for b in range(len(lengths)):
        L = lengths[b]
        if L == 0:
            firsts.append((7 * b + 1) % vocab)
            continue
        prompt = [(11 * b + 3 * i + 1) % vocab for i in range(L)]
        nxt = {g[b].prompt(prompt, 0) for g in groups}
        assert len(nxt) == 1
        firsts.append(nxt.pop())
    return firsts


def first_hits(ids):
    """Steps j whose id does not occur before j: a stop on ids[j] ends exactly at j."""
    return [j for j in range(len(ids)) if ids[j] not in ids[:j]]


def ragged_stops(full, vocab, b):
    """Member b's stop list over its probe's continuation `full`, by b mod 5: a stop on the first id; an id that never
    occurs (runs to max_steps); several ids, of which a middle one occurs first; none; a late first occurrence."""
    hits = first_hits(full)
    absent = next(t for t in range(vocab) if t not in full)
    kind = b % 5
    if kind == 0:
        return [full[0]]
    if kind == 1:
        return [absent]
    if kind == 2:
        j = hits[len(hits) // 2]
        return [absent, full[hits[-1]], full[j]]
    if kind == 3:
        return []
    return [full[hits[-1]]]


def expected(full, stops):
    return next((full[:j + 1] for j in range(len(full)) if full[j] in stops), full)


def assert_same_state(a, b, what, lp_exception=True):
    """a ran batch entries, b its own: logits, history, record and KV cache, all over the whole sequence."""
    assert_bit_equal(a.logits(), b.logits(), f"{what}: logits")
    assert np.array_equal(a.history(), b.history()), f"{what}: history"
    n = a.shape.seq_len
    for x, y, name in zip(a.logprobs(0, n), b.logprobs(0, n), ("ids", "lp", "top_ids", "top_lp")):
        if lp_exception and a.engine == "persistent" and name in ("lp", "top_lp"):
            # the megakernel sums the log-softmax normaliser from per-CTA partials, the chain's draw in
            # argmax_advance_kernel's order: the log-probabilities may differ in the last bits (DESIGN.md 5.14)
            np.testing.assert_allclose(x, y, rtol=2e-6, atol=0, err_msg=f"{what}: record {name}")
        else:
            assert_bit_equal(x, y, f"{what}: record {name}")
    for x, y in zip(a.kv_cache(), b.kv_cache()):
        assert_bit_equal(x, y, f"{what}: whole kv cache")


def until_vs_twins(members, twins, firsts, positions, max_steps, stops, what="", batch=None):
    """One Batch.generate_until against each twin's own generate_until; then each member's own generate continues
    from its end against its twin's.  Returns the ids and the stats."""
    own = batch is None
    batch = batch or Batch(members)
    got = [[] for _ in members]
    try:
        ids, stats = batch.generate_until(firsts, positions, max_steps, stops, on_tokens=lambda b, t: got[b].extend(t))
    finally:
        if own:
            batch.close()
    for b, (m, t) in enumerate(zip(members, twins)):
        assert got[b] == ids[b], f"{what} member {b}: callbacks"
        streamed = []
        assert t.generate_until(firsts[b], positions[b], max_steps[b], stops[b], on_tokens=streamed.extend) == ids[b], \
            f"{what} member {b}: ids"
        assert streamed == ids[b]
        assert_same_state(m, t, f"{what} member {b}")
    assert stats == {"passes": max(len(r) for r in ids), "rows": sum(len(r) for r in ids)}, what
    return ids, stats


def continue_own(members, twins, ids, positions, k, what):
    """Each member's own generate of k ids from where generate_until left it, against its twin's."""
    for b, (m, t) in enumerate(zip(members, twins)):
        p = positions[b] + len(ids[b])
        k_b = min(k, m.shape.seq_len - p)
        if k_b <= 0:
            continue
        assert m.generate(ids[b][-1], p, k_b) == t.generate(ids[b][-1], p, k_b), f"{what} member {b}: continued"
        assert_same_state(m, t, f"{what} member {b} continued")


def ragged_case(members, twins, probes, lengths, steps, what):
    """Stops of every kind (ragged_stops) from the probes' continuations, checked against the twins."""
    vocab = members[0].shape.vocab_size
    firsts = feed([members, twins, probes], lengths, vocab)
    stops = []
    for b, p in enumerate(probes):
        full = p.generate(firsts[b], lengths[b], steps[b])
        stops.append(ragged_stops(full, vocab, b))
        if b % 5 == 0:
            assert expected(full, stops[b]) == full[:1]
    ids, _ = until_vs_twins(members, twins, firsts, lengths, steps, stops, what)
    continue_own(members, twins, ids, lengths, 3, what)
    return ids


@pytest.mark.parametrize("key", ["hs16", "small", "hs128", "small-qwen", "small-int8"])
def test_ragged_stops_on_geometries(kllm_lib, engine, key):
    """B = 1, 3 and 8, members with prompts of different lengths: a stop on the first id, one never met, several
    ids, none, a late one."""
    shape = GEOMETRIES[key]
    for B in (1, 3, 8):
        members, twins, probes = trio(shape, engine, B)
        lengths = [min(2 + 9 * b, shape.seq_len // 4) for b in range(B)]
        steps = [[12, 9, 14, 7, 16, 10, 5, 13][b] for b in range(B)]
        if B == 1:
            steps = [10]
        ids = ragged_case(members, twins, probes, lengths, steps, f"{key} B={B}")
        if B == 8:
            assert len({len(r) for r in ids}) > 2, "the members did not end at different steps"
        for d in members + twins + probes:
            d.close()


def test_ragged_max_steps_without_stops(kllm_lib, engine):
    shape = SHAPES["small"]
    members, twins, _ = trio(shape, engine, MAX_BATCH)
    lengths = [3 * b for b in range(MAX_BATCH)]
    firsts = feed([members, twins], lengths, shape.vocab_size)
    steps = [16, 24, 32, 48, 4, 1, 40, 20]
    ids, stats = until_vs_twins(members, twins, firsts, lengths, steps, [[]] * MAX_BATCH, "ragged max_steps")
    assert [len(r) for r in ids] == steps
    assert stats == {"passes": 48, "rows": sum(steps)}


def test_equal_lengths_without_stops_equal_batch_generate(kllm_lib, engine):
    """generate_until with one length and no stops against kllm_batch_generate on a second member set."""
    shape = SHAPES["small"]
    members, others, _ = trio(shape, engine, 5)
    lengths = [1, 4, 9, 17, 30]
    firsts = feed([members, others], lengths, shape.vocab_size)
    a, b = Batch(members), Batch(others)
    ids, stats = a.generate_until(firsts, lengths, [20] * 5, [[]] * 5)
    assert b.generate(firsts, lengths, 20) == ids
    assert stats == {"passes": 20, "rows": 100}
    a.close(), b.close()
    for k, (m, o) in enumerate(zip(members, others)):
        assert_same_state(m, o, f"member {k}", lp_exception=False)


def test_each_member_draws_and_stops_under_its_own_settings(kllm_lib, engine):
    shape = SHAPES["small"]
    members, twins, probes = trio(shape, engine, MAX_BATCH, top_n=-1)
    for b in range(MAX_BATCH):
        for d in (members[b], twins[b], probes[b]):
            SETTINGS[b](d)
    lengths = [20 + b for b in range(MAX_BATCH)]
    steps = [24, 18, 30, 12, 26, 20, 16, 28]
    ids = ragged_case(members, twins, probes, lengths, steps, "settings")
    assert len({tuple(r) for r in ids}) > 1


def test_interleaved_with_own_entries_and_the_other_batch_calls(kllm_lib, engine):
    """generate_until in which member 0 stops first (so the running members move up a row), then the members' own
    entries, then kllm_batch_generate and kllm_batch_step on the same batch: the full table is back."""
    shape = SHAPES["small"]
    members, twins, probes = trio(shape, engine, 4)
    lengths = [5, 11, 2, 19]
    firsts = feed([members, twins, probes], lengths, shape.vocab_size)
    steps = [10, 14, 8, 12]
    full0 = probes[0].generate(firsts[0], lengths[0], steps[0])
    stops = [[full0[0]], [], [], []]
    batch = Batch(members)
    ids, _ = until_vs_twins(members, twins, firsts, lengths, steps, stops, "until", batch=batch)
    assert len(ids[0]) == 1 and [len(r) for r in ids[1:]] == steps[1:]
    pos = [lengths[b] + len(ids[b]) for b in range(4)]
    tok = [ids[b][-1] for b in range(4)]
    # the members' own entries
    for b in range(4):
        own = members[b].generate(tok[b], pos[b], 2)
        assert twins[b].generate(tok[b], pos[b], 2) == own
        tok[b], pos[b] = own[-1], pos[b] + 2
    # the batch's own calls, then generate_until once more
    got = batch.generate(tok, pos, 3)
    for b in range(4):
        assert twins[b].generate(tok[b], pos[b], 3) == got[b], f"generate member {b}"
        tok[b], pos[b] = got[b][-1], pos[b] + 3
    nxt = batch.step(tok, pos)
    for b in range(4):
        assert twins[b].step(tok[b], pos[b]) == nxt[b], f"step member {b}"
    tok, pos = nxt, [p + 1 for p in pos]
    for b in range(4):
        assert_same_state(members[b], twins[b], f"after generate and step, member {b}")
    until_vs_twins(members, twins, tok, pos, [3, 6, 1, 4], [[], [], [], []], "until again", batch=batch)
    batch.close()


@pytest.mark.parametrize("key,weight_format", [
    ("small-int8", "fp32"), ("small", "bf16"), ("small-qwen", "fp32"),
])
def test_weight_formats_and_shapes(kllm_lib, engine, key, weight_format):
    shape = replace(SHAPES[key], seq_len=min(SHAPES[key].seq_len, 256))
    members, twins, probes = trio(shape, engine, 5, weight_format)
    ragged_case(members, twins, probes, [2 + 5 * b for b in range(5)], [9, 6, 11, 4, 8], key)


@pytest.mark.parametrize("key", list(GRAPH_ONLY))
def test_graph_only_shapes(kllm_lib, monkeypatch, key):
    monkeypatch.setenv("KLLM_ENGINE", "graph")
    shape = GRAPH_ONLY[key]
    members, twins, probes = trio(shape, "graph", 4)
    S = shape.seq_len
    lengths = [0, 9, S - 300, S - 6]  # the cache's last rows, and members far apart
    ragged_case(members, twins, probes, lengths, [6, 5, 6, 6], key)


def test_refusals_leave_every_member_unchanged(kllm_lib, engine):
    shape = SHAPES["small"]
    S, V = shape.seq_len, shape.vocab_size
    w = synth_weights(shape, "cuda", 2024)
    a, b = Decoder(shape, w), Decoder(shape, w)
    if a.engine != engine:
        pytest.skip("engine")
    for d in (a, b):
        d.set_logprobs(2)
        d.generate(3, 0, 20)
    snaps = [snapshot(a), snapshot(b)]
    lib = a.lib
    batch = Batch([a, b])
    I32 = ctypes.c_int32

    def rc(first=(1, 2), pos=(20, 20), steps=(4, 4), stops=None, n_stop=(0, 1), null=None):
        stops = stops or [[], [7]]
        args = {"first": (I32 * 2)(*first), "pos": (I32 * 2)(*pos), "steps": (I32 * 2)(*steps),
                "stops": (I32 * (2 * MAX_STOP_IDS))(), "n_stop": (I32 * 2)(*n_stop), "out": (I32 * (2 * S))(),
                "n_out": (I32 * 2)()}
        for r, ids in enumerate(stops):
            for j, t in enumerate(ids):
                args["stops"][r * MAX_STOP_IDS + j] = t
        if null:
            args[null] = None
        return lib.kllm_batch_generate_until(batch.handle, args["first"], args["pos"], args["steps"], args["stops"],
                                             args["n_stop"], BATCH_TOKEN_CALLBACK(), None, args["out"], args["n_out"],
                                             ctypes.byref(BatchStats()))

    for null in ("first", "pos", "steps", "stops", "n_stop", "out", "n_out"):
        assert rc(null=null) == E_INVALID, null
    bad = [
        dict(steps=(4, 0)), dict(steps=(-2, 4)),  # max_steps <= 0
        dict(pos=(-1, 20)),  # start < 0
        dict(pos=(20, S - 3)), dict(steps=(S - 19, 4)),  # start + max_steps > seq_len
        dict(n_stop=(0, MAX_STOP_IDS + 1)), dict(n_stop=(-1, 1)),  # n_stop outside [0, KLLM_MAX_STOP_IDS]
        dict(stops=[[], [V]]), dict(stops=[[], [-1]]), dict(stops=[[5, V], []], n_stop=(2, 0)),  # stop id
        dict(first=(V, 2)), dict(first=(1, -1)),  # first token outside [0, vocab)
    ]
    for kw in bad:
        assert rc(**kw) == E_INVALID, kw
    I = (I32 * 2)(1, 2)
    assert lib.kllm_batch_generate_until(None, I, I, I, (I32 * 32)(), (I32 * 2)(), BATCH_TOKEN_CALLBACK(), None,
                                         (I32 * 64)(), (I32 * 2)(), None) == E_INVALID
    batch.close()
    for d, snap, name in ((a, snaps[0], "a"), (b, snaps[1], "b")):
        assert_unchanged(d, snap, f"member {name} after the refusals")
    # a stop id at the edge of the vocabulary and a full stop list are accepted
    batch = Batch([a, b])
    assert rc(stops=[[V - 1], list(range(MAX_STOP_IDS))], n_stop=(1, MAX_STOP_IDS), steps=(2, 2)) == 0
    batch.close()


def test_callbacks(kllm_lib, engine):
    """A NULL callback works; an exception raised in a Python callback is re-raised after the call, and every member
    still ends as its twin."""
    shape = SHAPES["small"]
    members, twins, probes = trio(shape, engine, 3)
    lengths = [4, 8, 12]
    firsts = feed([members, twins, probes], lengths, shape.vocab_size)
    steps = [6, 9, 5]
    full = [p.generate(firsts[b], lengths[b], steps[b]) for b, p in enumerate(probes)]
    stops = [[full[0][3]] if full[0][3] not in full[0][:3] else [], [], [full[2][0]]]
    batch = Batch(members)
    ids, stats = batch.generate_until(firsts, lengths, steps, stops)  # no callback
    for b in range(3):
        assert ids[b] == expected(full[b], stops[b])
        assert twins[b].generate_until(firsts[b], lengths[b], steps[b], stops[b]) == ids[b]
        assert_same_state(members[b], twins[b], f"no callback, member {b}")
    # again from the same positions, with a callback that raises at its second call
    calls = []

    def boom(member, t):
        calls.append((member, t))
        if len(calls) == 2:
            raise ValueError("from the callback")

    with pytest.raises(ValueError, match="from the callback"):
        batch.generate_until(firsts, lengths, steps, stops, on_tokens=boom)
    batch.close()
    assert sum(len(t) for _, t in calls) == sum(len(r) for r in ids), "the loop ran to its end"
    for b in range(3):
        assert [i for m, t in calls if m == b for i in t] == ids[b]
        assert_same_state(members[b], twins[b], f"after the raising callback, member {b}")
