"""-m gpu: kllm_batch_beam_search against twin decoders, bit for bit.  The twins are 2 B decoders over the same weights
on the same engine, in two ping-pong sets forked with copy_prefix: each pass they step every beam's sequence on their
own, and kllm_logprobs_f32 over their logits gives the candidates that kuiperllama_b200/beam.py runs the rule over.
Also: B = 1 against greedy generate_until, the best hypothesis against Decoder.score, the prompt copy, the refusals,
and the batch's other entries afterwards."""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import GEOMETRIES
from gpu_util import assert_bit_equal, ptr
from kuiperllama_b200 import SHAPES, Batch, Decoder, KllmError, check, sampling, synth_weights
from kuiperllama_b200 import beam
from kuiperllama_b200.decoder import bf16_weights

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -2

GRAPH_ONLY_HS256 = replace(SHAPES["small"], name="hs256", dim=512, hidden_dim=1376, layer_num=2, head_num=2,
                           kv_head_num=1, vocab_size=1024, seq_len=544)  # head_size 256: the graph engine only


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def make(shape, engine, n, weight_format="fp32", seed=77):
    w = synth_weights(shape, "cuda", seed)
    if weight_format == "bf16":
        w = bf16_weights(w)
    try:
        ds = [Decoder(shape, w, weight_format=weight_format) for _ in range(n)]
    except KllmError:
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    if ds[0].engine != engine:
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    for d in ds:
        d.set_logprobs(3)  # the record setting does not matter to the search
    return ds


def top_candidates(d, top_n):
    """kllm_logprobs_f32 over the decoder's logits: its top_n ids and their lp"""
    lib, V = d.lib, d.shape.vocab_size
    ids = torch.zeros(1, dtype=torch.int32, device="cuda")
    lp = torch.empty(1, device="cuda")
    ti = torch.empty(top_n, dtype=torch.int32, device="cuda")
    tl = torch.empty(top_n, device="cuda")
    check(lib.kllm_logprobs_f32(ctypes.c_void_p(lib.kllm_decoder_logits_device(d.handle)), V, ptr(ids), 1, top_n,
                                ptr(lp), ptr(ti), ptr(tl), None), "kllm_logprobs_f32")
    torch.cuda.synchronize()
    return [int(i) for i in ti.cpu().numpy()], tl.cpu().numpy()


def twin_search(sets, B, first, start, max_new, eos, alpha, early, n_return):
    """beam.py over the twins: sets[0][0] holds the prompt; pass p forks beam j's twin from its parent's"""
    state = list(sets)
    top = B + len(eos)

    def candidates(beams):
        p = len(beams[0].ids)
        if p == 0:
            state[0][0].step(first, start)
            return [top_candidates(state[0][0], top)]
        cur, nxt = state
        out = []
        for j, bm in enumerate(beams):
            nxt[j].copy_prefix(cur[bm.parent], start + p)
            nxt[j].step(bm.ids[-1], start + p)
            out.append(top_candidates(nxt[j], top))
        state[0], state[1] = nxt, cur
        return out

    return beam.beam_search(candidates, B, max_new, eos, alpha, early, n_return, start)


def prompt_of(n, vocab):
    return [(13 * i + 5) % vocab for i in range(n)]


def prefill(ds, start, vocab):
    """ds hold the same prompt of `start` ids; returns the id fed at start"""
    if start == 0:
        return 11 % vocab
    nxt = [d.prompt(prompt_of(start, vocab), 0) for d in ds]
    assert len(set(nxt)) == 1
    return nxt[0]


def greedy_eos(d, first, start, n_eos, max_new):
    """eos ids from a greedy continuation, as tools/bench_batch_until.py picks stops, so that beams finish early"""
    if n_eos == 0:
        return []
    ids = d.generate(first, start, max(max_new, 2 * n_eos + 2))
    picks = []
    for i in ids[1::2]:
        if i not in picks:
            picks.append(i)
    return picks[:n_eos]


def run_case(shape, engine, weight_format, B, start, max_new, n_eos, alpha, early):
    ds = make(shape, engine, 3 * B, weight_format)
    members, sets = ds[:B], (ds[B:2 * B], ds[2 * B:])
    V = shape.vocab_size
    first = prefill([members[0], sets[0][0], sets[1][0]], start, V)
    eos = greedy_eos(sets[1][0], first, start, n_eos, max_new)
    k0, v0 = members[0].kv_cache()
    batch = Batch(members)
    try:
        hyps, stats = batch.beam_search(first, start, max_new, eos, alpha, early, n_return=B)
        want, wstats = twin_search(sets, B, first, start, max_new, eos, alpha, early, B)
        assert stats == wstats
        assert len(hyps) == B
        for i, (h, w) in enumerate(zip(hyps, want)):
            assert h["ids"] == w["ids"], i
            assert np.float32(h["score"]).view(np.uint32) == np.float32(w["score"]).view(np.uint32), (i, h, w)
            assert np.float32(h["sum"]).view(np.uint32) == np.float32(w["sum"]).view(np.uint32), (i, h, w)
        # member 0's prompt rows are unchanged and every member holds them
        k, v = members[0].kv_cache()
        assert_bit_equal(k[:, :start], k0[:, :start], "member 0 keys")
        assert_bit_equal(v[:, :start], v0[:, :start], "member 0 values")
        for b, m in enumerate(members[1:], 1):
            kb, vb = m.kv_cache()
            assert_bit_equal(kb[:, :start + 1], k[:, :start + 1], f"member {b} keys")
            assert_bit_equal(vb[:, :start + 1], v[:, :start + 1], f"member {b} values")
        # the batch's other entries afterwards, against the twins
        firsts, zeros = [3 + b for b in range(B)], [0] * B
        ids = batch.generate(firsts, zeros, 4)
        for b in range(B):
            assert sets[0][b].generate(firsts[b], 0, 4) == ids[b], b
            assert_bit_equal(members[b].logits(), sets[0][b].logits(), f"generate member {b}")
        ids, _ = batch.generate_until(firsts, [4] * B, [3] * B, [[]] * B)
        for b in range(B):
            assert sets[0][b].generate_until(firsts[b], 4, 3) == ids[b], b
    finally:
        batch.close()
    return hyps, stats, eos


CASES = [
    # key, weight format, B, start, max_new, n_eos, length penalty, early stopping
    ("small", "fp32", 3, 40, 12, 2, 1.0, False),
    ("small", "bf16", 8, 0, 10, 2, 2.0, "never"),
    ("small-int8", "fp32", 2, 20, 8, 1, -0.5, True),
    ("small-qwen", "fp32", 8, 30, 6, 3, 0.0, False),
    ("gqa", "fp32", 3, 100, 9, 1, 1.0, "never"),
    ("end", "fp32", 2, 150, 10, 0, 1.0, False),  # start + max_new = seq_len
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-{c[1]}-B{c[2]}" for c in CASES])
def test_beam_search_equals_twins(kllm_lib, engine, case):
    key, wf, B, start, max_new, n_eos, alpha, early = case
    if key == "gqa":
        shape = replace(GEOMETRIES["gqa-hs64"], seq_len=256)
    elif key == "end":
        shape = replace(SHAPES["small"], seq_len=start + max_new)
    else:
        shape = replace(SHAPES[key], seq_len=min(SHAPES[key].seq_len, 256))
    hyps, stats, eos = run_case(shape, engine, wf, B, start, max_new, n_eos, alpha, early)
    assert stats["passes"] >= 1


def test_graph_only_shape(kllm_lib, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", "graph")
    run_case(GRAPH_ONLY_HS256, "graph", "fp32", 3, 500, 12, 1, 1.0, False)


def test_one_beam_is_greedy(kllm_lib, engine):
    """B = 1 with length penalty 0: a next beam never scores above the eos that ranked before it, so the search stops
    at the first eos, as generate_until does; S is the sum of the record's lp"""
    shape = replace(SHAPES["small"], seq_len=256)
    m, twin = make(shape, engine, 2)
    start = 30
    first = prefill([m, twin], start, shape.vocab_size)
    eos = greedy_eos(twin, first, start, 2, 20)
    twin.set_logprobs(0)
    batch = Batch([m])
    try:
        hyps, stats = batch.beam_search(first, start, 20, eos, 0.0, False)
    finally:
        batch.close()
    ids = twin.generate_until(first, start, 20, eos)
    assert hyps[0]["ids"] == ids
    assert stats == {"passes": len(ids), "forks": 0, "fork_rows": 0}
    _, lp, _, _ = twin.logprobs(start, len(ids))
    s = np.float32(0)
    for x in lp:
        s = np.float32(s + x)
    if engine == "graph":
        assert np.float32(hyps[0]["sum"]).view(np.uint32) == s.view(np.uint32)
    else:  # the record's lp come from the megakernel's partition (DESIGN.md 5.14)
        np.testing.assert_allclose(hyps[0]["sum"], s, rtol=2e-6, atol=0)


def test_best_sum_is_the_models_score(kllm_lib, engine):
    shape = replace(SHAPES["small"], seq_len=256)
    ds = make(shape, engine, 5)
    start, V = 25, shape.vocab_size
    first = prefill(ds[:1], start, V)
    batch = Batch(ds[:4])
    try:
        hyps, _ = batch.beam_search(first, start, 12, [], 1.0, False)
    finally:
        batch.close()
    ids = hyps[0]["ids"]
    lp = ds[4].score(prompt_of(start, V) + [first] + ids, 0)[-len(ids):]
    k = sampling.chain_persistent(V, 132 * 4) + sampling.chain_one_block(V)
    bound = 2 * float(np.sum(sampling.logprob_bound(lp, k, V))) + len(ids) * 2.0 ** -24 * abs(float(np.sum(lp)))
    assert abs(float(hyps[0]["sum"]) - float(np.sum(lp.astype(np.float64)))) <= bound


def test_refusals_leave_every_member_unchanged(kllm_lib, engine):
    shape = replace(SHAPES["small"], seq_len=128)
    S, V = shape.seq_len, shape.vocab_size
    ds = make(shape, engine, 3)
    for d in ds:
        d.generate(3, 0, 20)
    snaps = [(d.logits(), d.history(), d.kv_cache()) for d in ds]
    batch = Batch(ds)
    lib, h = batch.lib, batch.handle
    ids, lens = (ctypes.c_int32 * 64)(), (ctypes.c_int32 * 3)()
    sc, sm = (ctypes.c_float * 3)(), (ctypes.c_float * 3)()
    eos = (ctypes.c_int32 * 9)(*range(1, 10))

    def rc(first=5, start=10, max_new=4, e=eos, n_eos=1, alpha=1.0, early=0, n_ret=1, out=(ids, lens, sc, sm)):
        return lib.kllm_batch_beam_search(h, first, start, max_new, e, n_eos, alpha, early, n_ret, *out, None)

    invalid = [dict(out=(None, lens, sc, sm)), dict(out=(ids, None, sc, sm)), dict(out=(ids, lens, None, sm)),
               dict(out=(ids, lens, sc, None)), dict(first=-1), dict(first=V), dict(start=-1), dict(max_new=0),
               dict(start=S - 3, max_new=4), dict(n_eos=-1), dict(n_eos=9), dict(e=None, n_eos=1),
               dict(e=(ctypes.c_int32 * 1)(V)), dict(e=(ctypes.c_int32 * 1)(-1)), dict(n_ret=0), dict(n_ret=4),
               dict(alpha=float("inf")), dict(alpha=float("nan")), dict(early=-1), dict(early=3)]
    for kw in invalid:
        assert rc(**kw) == E_INVALID, kw
    assert lib.kllm_batch_beam_search(None, 5, 10, 4, eos, 1, 1.0, 0, 1, ids, lens, sc, sm, None) == E_INVALID
    for setting in (lambda d: d.set_sampling(0.7, 10, 3), lambda d: d.set_repetition_penalty(1.2),
                    lambda d: d.set_frequency_presence(0.5, 0.0), lambda d: d.set_frequency_presence(0.0, 0.5),
                    lambda d: d.set_logit_bias({4: 1.0})):
        setting(ds[2])
        assert rc() == E_UNSUPPORTED
        ds[2].set_sampling(0.0), ds[2].set_repetition_penalty(1.0), ds[2].set_frequency_presence(0.0, 0.0)
        ds[2].set_logit_bias(None)
    batch.close()
    for d, (logits, hist, kv) in zip(ds, snaps):
        assert_bit_equal(d.logits(), logits, "logits")
        assert np.array_equal(d.history(), hist), "history"
        for x, y in zip(d.kv_cache(), kv):
            assert_bit_equal(x, y, "cache")
    # K = max(2, 1 + n_eos) * B over 8 members of a 40-id vocabulary: 40 with four eos ids, 48 > 40 with five
    vs = make(replace(shape, vocab_size=40), engine, 8)
    vb = Batch(vs)
    snap = vs[3].kv_cache()
    assert vb.lib.kllm_batch_beam_search(vb.handle, 5, 10, 4, eos, 5, 1.0, 0, 1, ids, lens, sc, sm, None) == \
        E_UNSUPPORTED
    vb.close()
    for x, y in zip(vs[3].kv_cache(), snap):
        assert_bit_equal(x, y, "cache")
