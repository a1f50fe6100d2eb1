"""-m gpu: speculative decoding -- kllm_decoder_verify against kllm_decoder_generate of the accepted length on a twin
decoder over the same weights, and kllm_decoder_generate_speculative against kllm_decoder_generate_until, bit for bit:
ids, logits, history, log-probability record and the KV rows up to the frontier."""
import ctypes
from dataclasses import replace

import numpy as np
import pytest

from decode_model_util import GEOMETRIES
from gpu_util import assert_bit_equal
from kuiperllama_b200 import SHAPES, Decoder, KllmError, ModelShape, synth_weights
from kuiperllama_b200.decoder import bf16_weights
from kuiperllama_b200.speculative import lookup_draft, simulate_rounds

pytestmark = pytest.mark.gpu

# shapes only the graph engine takes: head_size 256, int8 scale rows of 36 bytes, seq_len % 4 != 0
GRAPH_ONLY = {
    "hs256": ModelShape("hs256", 512, 1376, 2, 2, 1, 1024, 544),
    "int8-g32-hs48": ModelShape("int8-g32-hs48", 288, 768, 2, 6, 2, 1024, 544, group_size=32),
    "seq1001": replace(SHAPES["small"], name="small-seq1001", seq_len=1001),
}


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def twins(shape, engine, weight_format="fp32", seed=2024):
    w = synth_weights(shape, "cuda", seed)
    if weight_format == "bf16":
        w = bf16_weights(w)
    try:
        a, b = Decoder(shape, w, weight_format=weight_format), Decoder(shape, w, weight_format=weight_format)
    except KllmError:
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    if a.engine != engine:
        a.close(), b.close()
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    return a, b


def assert_same_state(a, b, upto, what):
    assert_bit_equal(a.logits(), b.logits(), f"{what}: logits")
    assert np.array_equal(a.history(), b.history()), f"{what}: history"
    n = a.shape.seq_len
    for x, y, name in zip(a.logprobs(0, n), b.logprobs(0, n), ("ids", "lp", "top_ids", "top_lp")):
        if a.engine == "persistent" and name in ("lp", "top_lp"):
            # the megakernel sums the log-softmax normaliser from per-CTA partials; the verify pass sums it in
            # argmax_advance_kernel's order, so the log-probabilities may differ in the last bits (DESIGN.md 5.13)
            np.testing.assert_allclose(x, y, rtol=2e-6, atol=0, err_msg=f"{what}: record {name}")
        else:
            assert_bit_equal(x, y, f"{what}: record {name}")
    for x, y in zip(a.kv_cache(), b.kv_cache()):
        assert_bit_equal(x[:, :upto], y[:, :upto], f"{what}: kv rows")


def sweep(a, b, first, p, lengths=range(1, 9)):
    """Every verify length n and every cut a: drafts from a reference run with the id at a + 1 altered."""
    vocab = a.shape.vocab_size
    cont = a.generate(first, p, 8)
    assert b.generate(first, p, 8) == cont
    for n in lengths:
        for cut in range(n):
            drafts = list(cont[:n - 1])
            if cut < n - 1:
                drafts[cut] = (drafts[cut] + 1) % vocab
            ids = a.verify([first] + drafts, p)
            assert ids == cont[:cut + 1], (n, cut)
            assert b.generate(first, p, cut + 1) == ids
            assert_same_state(a, b, p + cut + 1, f"n={n} a={cut}")


@pytest.mark.parametrize("key", list(GEOMETRIES))
def test_verify_matches_generate_on_every_geometry(kllm_lib, engine, key):
    shape = GEOMETRIES[key]
    a, b = twins(shape, engine)
    a.set_logprobs(5), b.set_logprobs(5)
    p = min(40, shape.seq_len - 9)
    a.generate(3, 0, p), b.generate(3, 0, p)
    lengths = range(1, 9) if shape.layer_num * shape.dim <= 2048 * 4 else (1, 4, 8)
    sweep(a, b, 5, p, lengths)


@pytest.mark.parametrize("key", list(GRAPH_ONLY))
def test_verify_on_graph_only_shapes(kllm_lib, monkeypatch, key):
    monkeypatch.setenv("KLLM_ENGINE", "graph")
    shape = GRAPH_ONLY[key]
    a, b = twins(shape, "graph")
    p = shape.seq_len - 9  # the cache's last rows
    sweep(a, b, 7, p, (1, 3, 8))


@pytest.mark.parametrize("name", ["small", "tinyllama-1.1b"])
def test_verify_bf16_weights(kllm_lib, engine, name):
    shape = replace(SHAPES[name], seq_len=256)
    a, b = twins(shape, engine, "bf16")
    a.generate(2, 0, 30), b.generate(2, 0, 30)
    sweep(a, b, 9, 30, (1, 2, 5, 8))


def test_verify_over_a_rewound_prefix(kllm_lib, engine):
    a, b = twins(SHAPES["small"], engine)
    a.generate(4, 0, 120), b.generate(4, 0, 120)  # a longer earlier run leaves rows past the rewind point
    sweep(a, b, 11, 50)


SETTINGS = {
    "sampling": lambda d: d.set_sampling(0.8, 40, 1234, top_p=0.9),
    "repetition": lambda d: d.set_repetition_penalty(1.3, 16),
    "freq-presence": lambda d: d.set_frequency_presence(0.5, 0.4, 20),
    "logit-bias": lambda d: d.set_logit_bias({5: 3.0, 17: -100.0, 42: 2.5}),
    "all": lambda d: (d.set_sampling(1.1, 0, 2**40 + 3), d.set_repetition_penalty(0.8, 0),
                      d.set_frequency_presence(-0.3, 0.2, 0), d.set_logit_bias({9: 4.0})),
}


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_verify_under_each_draw_setting(kllm_lib, engine, setting):
    a, b = twins(SHAPES["small"], engine)
    for d in (a, b):
        SETTINGS[setting](d)
        d.set_logprobs(5)
        d.generate(3, 0, 30)
    sweep(a, b, 6, 30)


def spec_vs_until(a, b, first, p, max_steps, stops=(), draft_len=4, ngram_max=3):
    ctx = [int(t) for t in b.history()[:p]] + [first]
    got = []
    ids, stats = a.generate_speculative(first, p, max_steps, stops, on_tokens=got.extend, draft_len=draft_len,
                                        ngram_max=ngram_max)
    ref = b.generate_until(first, p, max_steps, stops)
    assert ids == ref and got == ids
    assert_same_state(a, b, p + len(ids), f"speculative from {p}")
    assert stats == simulate_rounds(ctx, ids, draft_len=draft_len, ngram_max=ngram_max, max_steps=max_steps,
                                    seq_len=a.shape.seq_len, stop_ids=stops)
    return ids, stats


def inside_rounds(context, ids, draft_len, ngram_max, max_steps, seq_len):
    """The indices of the ids a verify round drew after its first id (kllm_b200.h's round structure)."""
    c, produced, inner = list(context), 0, []
    while produced < len(ids):
        m = min(draft_len, max_steps - produced - 1, seq_len - (len(context) - 1 + produced) - 1)
        draft = lookup_draft(c, ngram_max, m)
        a = 0
        while a < len(draft) and produced + a < len(ids) and draft[a] == ids[produced + a]:
            a += 1
        inner += range(produced + 1, produced + a + 1)
        c += ids[produced:produced + a + 1]
        produced += a + 1
    return inner


def test_generate_speculative_matches_generate_until(kllm_lib, engine):
    shape = replace(SHAPES["small"], seq_len=512)
    a, b = twins(shape, engine)
    a.set_logprobs(3), b.set_logprobs(3)
    prompt = [7, 8, 9, 10, 11, 7, 8, 9, 10, 11, 7, 8, 9]  # repetitive: the lookup finds drafts
    assert a.prompt(prompt, 0) == b.prompt(prompt, 0)
    p, first = len(prompt), prompt[-1]
    total = 0
    for draft_len in (1, 3, 7):
        ids, stats = spec_vs_until(a, b, first, p, 120, draft_len=draft_len)
        total += stats["accepted"]
    assert total > 0, "no fixed workload accepted a draft"
    # a stop id inside a round, max_steps inside a round, a start near seq_len
    ids, _ = spec_vs_until(a, b, first, p, 120)
    ctx = [int(t) for t in b.history()[:p]] + [first]
    inner = [j for j in inside_rounds(ctx, ids, 4, 3, 120, shape.seq_len) if ids[j] not in ids[:j]]
    assert inner, "no id is drawn inside a verify round past its first"
    spec_vs_until(a, b, first, p, 120, stops=[ids[inner[0]]])
    for m in (1, 2, 5, 23):
        spec_vs_until(a, b, first, p, m)
    near = shape.seq_len - 6
    a.generate(first, p, near - p), b.generate(first, p, near - p)
    spec_vs_until(a, b, 3, near, 6, draft_len=7, ngram_max=8)


def test_generate_speculative_on_its_own_greedy_continuation(kllm_lib, engine):
    a, b = twins(replace(SHAPES["tinyllama-1.1b"], seq_len=512), engine)
    first = 1
    cont = a.generate(first, 0, 64)
    b.generate(first, 0, 64)
    # feed the continuation again, so that the lookup finds drafts in its first copy
    a.prompt([first] + cont, 64), b.prompt([first] + cont, 64)
    spec_vs_until(a, b, cont[-1], 129, 100, draft_len=7)


def test_draft_decoder_beside_its_target(kllm_lib, engine):
    """A small draft model proposes with generate, the target checks with verify, the draft rewinds."""
    target_shape = replace(SHAPES["small"], seq_len=256)
    draft_shape = replace(SHAPES["tiny"], vocab_size=target_shape.vocab_size, seq_len=256)
    target, ref = twins(target_shape, engine)
    draft = Decoder(draft_shape, synth_weights(draft_shape, "cuda", 77))
    first, p, out, K = 5, 0, [], 4
    while len(out) < 60:
        k = min(K, 60 - len(out) - 1)
        proposal = draft.generate(first, p, k) if k > 0 else []
        ids = target.verify([first] + proposal, p)
        out += ids
        p += len(ids)
        first = ids[-1]
        # the draft rewinds: its rows past p are fed again by the next round
    assert out == ref.generate_until(5, 0, 60)


def test_refusals_leave_the_decoder_unchanged(kllm_lib, engine):
    shape = SHAPES["small"]
    a, b = twins(shape, engine)
    a.set_logprobs(2), b.set_logprobs(2)
    a.generate(3, 0, 20), b.generate(3, 0, 20)
    S, V = shape.seq_len, shape.vocab_size
    bad = [([], 5), ([1] * 9, 5), ([1, -1], 5), ([1, V], 5), ([1, 2], -1), ([1, 2, 3], S - 2)]
    for tokens, p in bad:
        with pytest.raises(KllmError):
            a.verify(tokens, p)
        assert_same_state(a, b, S, f"refused verify {tokens} at {p}")
    for kw in ({"draft_len": 0}, {"draft_len": 8}, {"ngram_max": 0}, {"ngram_max": 9}):
        with pytest.raises(KllmError):
            a.generate_speculative(3, 20, 10, **kw)
        assert_same_state(a, b, S, f"refused speculative {kw}")


def test_fast_numerics_are_refused(kllm_lib, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", "persistent")
    shape = SHAPES["small"]
    w = synth_weights(shape, "cuda", 5)
    a = Decoder(shape, w, numerics="fast")
    a.generate(3, 0, 10)
    before = (a.logits(), a.history())
    assert a.lib.kllm_decoder_verify(a.handle, (ctypes.c_int32 * 2)(1, 2), 2, 10, (ctypes.c_int32 * 2)(),
                                     ctypes.byref(ctypes.c_int32())) == -2  # KLLM_E_UNSUPPORTED
    with pytest.raises(KllmError):
        a.generate_speculative(3, 10, 5)
    assert_bit_equal(a.logits(), before[0], "logits after a refusal")
    assert np.array_equal(a.history(), before[1])
    # the bf16 KV cache needs the fast numerics: refused as well
    c = Decoder(shape, w, numerics="fast", kv_cache="bf16")
    assert c.lib.kllm_decoder_verify(c.handle, (ctypes.c_int32 * 2)(1, 2), 2, 0, (ctypes.c_int32 * 2)(),
                                     ctypes.byref(ctypes.c_int32())) == -2


def test_null_pointers_are_refused(kllm_lib, engine):
    a, _ = twins(SHAPES["small"], engine)
    toks, out, n = (ctypes.c_int32 * 2)(1, 2), (ctypes.c_int32 * 2)(), ctypes.c_int32()
    lib = a.lib
    assert lib.kllm_decoder_verify(None, toks, 2, 0, out, ctypes.byref(n)) == -1
    assert lib.kllm_decoder_verify(a.handle, None, 2, 0, out, ctypes.byref(n)) == -1
    assert lib.kllm_decoder_verify(a.handle, toks, 2, 0, None, ctypes.byref(n)) == -1
    assert lib.kllm_decoder_verify(a.handle, toks, 2, 0, out, None) == -1
    from kuiperllama_b200 import TOKEN_CALLBACK
    outs = (ctypes.c_int32 * 8)()
    assert lib.kllm_decoder_generate_speculative(a.handle, 1, 0, 8, None, 0, 2, 3, TOKEN_CALLBACK(), None, None,
                                                 ctypes.byref(n), None) == -1
    assert lib.kllm_decoder_generate_speculative(a.handle, 1, 0, 8, None, 1, 2, 3, TOKEN_CALLBACK(), None, outs,
                                                 ctypes.byref(n), None) == -1
