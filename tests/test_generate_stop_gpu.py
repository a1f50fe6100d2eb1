"""-m gpu: kllm_decoder_generate_until on both engines -- the stop on the device (persistent) or between host-driven
steps (graph), the ids streamed while the loop runs, and the state it leaves behind, checked bit for bit against
kllm_decoder_generate on a second decoder over the same weights."""
import ctypes
import random
import time

import numpy as np
import pytest

from gpu_util import assert_bit_equal
from kuiperllama_b200 import SHAPES, Decoder, load_library, synth_weights

pytestmark = pytest.mark.gpu

PROMPT = [1, 7, 3, 12, 5]
SAMPLING = [None, (0.8, 40, 1234), (0.9, 0, 2**40 + 9)]


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def pair(name, numerics, engine):
    """Two decoders over the same weights: the one under test and the reference."""
    shape = SHAPES[name]
    w = synth_weights(shape, "cuda", 2024)
    a, b = Decoder(shape, w, numerics=numerics), Decoder(shape, w, numerics=numerics)
    if engine == "persistent" and a.engine != "persistent":
        pytest.skip(f"{name}: the persistent engine does not take this shape")
    assert a.engine == b.engine == engine
    return shape, a, b


def until(dec, first, pos, max_steps, stops=()):
    """generate_until with a recording callback; the callbacks' concatenation must equal the result."""
    got = []
    ids = dec.generate_until(first, pos, max_steps, stops, on_tokens=got.extend)
    assert got == ids
    return ids


def first_hits(ids):
    """Steps j whose id does not occur before j: a stop on ids[j] ends exactly at j."""
    return [j for j in range(len(ids)) if ids[j] not in ids[:j]]


def kv_rows(dec, n):
    k, v = dec.kv_cache()
    return k[:, :n], v[:, :n]


def check_stops(shape, dut, ref, first, sp, M):
    full = ref.generate(first, sp, M)
    full_logits = ref.logits()
    # no stop ids: ids, logits and KV cache bit-identical to generate(max_steps)
    assert until(dut, first, sp, M) == full
    assert_bit_equal(dut.logits(), full_logits, "logits, no stop")
    for a, b in zip(kv_rows(dut, sp + M), kv_rows(ref, sp + M)):
        assert_bit_equal(a, b, "kv, no stop")
    absent = next(t for t in range(shape.vocab_size) if t not in full)
    assert until(dut, first, sp, M, [absent]) == full
    hits = first_hits(full)
    js = sorted({hits[0], hits[len(hits) // 2], hits[-1]})  # step 0, a middle step, the last first occurrence
    assert hits[0] == 0
    for j in js:
        ids = until(dut, first, sp, M, [full[j]])
        assert ids == full[:j + 1], j
        ref.generate(first, sp, j + 1)
        assert_bit_equal(dut.logits(), ref.logits(), f"logits after a stop at {j}")
        for a, b in zip(kv_rows(dut, sp + j + 1), kv_rows(ref, sp + j + 1)):
            assert_bit_equal(a, b, f"kv after a stop at {j}")
        # resume where the stop left off: the uninterrupted run continues bit for bit
        if j + 1 < M:
            assert dut.generate(full[j], sp + j + 1, M - j - 1) == full[j + 1:], j
            ref.generate(first, sp, M)
            assert_bit_equal(dut.logits(), ref.logits(), f"logits after resuming at {j + 1}")
    # several stop ids at once: the first one that occurs ends the run
    j = js[len(js) // 2]
    assert until(dut, first, sp, M, [absent, full[js[-1]], full[j]]) == full[:j + 1]
    if M - 1 in hits:  # a stop on the very last step
        assert until(dut, first, sp, M, [full[M - 1]]) == full


@pytest.mark.parametrize("numerics", ["exact", "fast"])
@pytest.mark.parametrize("name", ["small", "small-int8", "small-qwen"])
def test_stop_matches_generate(engine, name, numerics):
    shape, dut, ref = pair(name, numerics, engine)
    for s in SAMPLING:
        for d in (dut, ref):
            d.set_sampling(*(s or (0.0, 0, 0)))
        first = dut.prompt(PROMPT)
        assert ref.prompt(PROMPT) == first
        check_stops(shape, dut, ref, first, len(PROMPT), 40)
        # start_pos + max_steps == seq_len
        M = 24
        sp = shape.seq_len - M
        first = dut.prompt([3, 1, 4], sp - 3)
        assert ref.prompt([3, 1, 4], sp - 3) == first
        check_stops(shape, dut, ref, first, sp, M)


@pytest.mark.parametrize("name", ["small", "small-qwen"])
def test_mixed_calls_keep_the_engine_in_step(engine, name):
    """30 calls of generate_until (with and without a hit), generate, step and prompt on one decoder match a
    second decoder that only runs generate / step / prompt: the persistent engine's tags and barrier counts
    follow the positions that ran, not max_steps."""
    shape, dut, ref = pair(name, "exact", engine)
    rng = random.Random(5)
    for s in (None, (0.8, 40, 77)):
        for d in (dut, ref):
            d.set_sampling(*(s or (0.0, 0, 0)))
        tok = dut.prompt(PROMPT)
        assert ref.prompt(PROMPT) == tok
        pos = len(PROMPT)
        for call in range(30):
            room = shape.seq_len - pos
            if room < 8:
                tok = dut.prompt(PROMPT)
                assert ref.prompt(PROMPT) == tok
                pos = len(PROMPT)
                continue
            op = ("until", "generate", "step", "prompt")[call % 4]
            if op == "until":
                M = rng.randint(1, min(20, room))
                probe = ref.generate(tok, pos, M)
                stops = [probe[rng.randrange(M)]] if call % 8 == 0 else [rng.randrange(shape.vocab_size)]
                ids = until(dut, tok, pos, M, stops)
                want = next((probe[:j + 1] for j in range(M) if probe[j] in stops), probe)
                assert ids == want, call
                ref.generate(tok, pos, len(ids))
                tok, pos = ids[-1], pos + len(ids)
            elif op == "generate":
                M = rng.randint(1, min(6, room))
                ids = dut.generate(tok, pos, M)
                assert ref.generate(tok, pos, M) == ids, call
                tok, pos = ids[-1], pos + M
            elif op == "step":
                nxt = dut.step(tok, pos)
                assert ref.step(tok, pos) == nxt, call
                tok, pos = nxt, pos + 1
            else:
                p = [rng.randrange(shape.vocab_size) for _ in range(3)]
                nxt = dut.prompt(p, pos)
                assert ref.prompt(p, pos) == nxt, call
                tok, pos = nxt, pos + 3
            assert_bit_equal(dut.logits(), ref.logits(), f"logits after call {call} ({op})")
        for a, b in zip(kv_rows(dut, pos), kv_rows(ref, pos)):
            assert_bit_equal(a, b, "kv after the mixed calls")


def test_invalid_arguments_touch_nothing(engine):
    shape, dut, _ = pair("small", "exact", engine)
    lib = load_library()
    first = dut.prompt(PROMPT)
    k0, v0 = dut.kv_cache()
    lg0 = dut.logits()
    I32 = ctypes.c_int32
    out = (I32 * shape.seq_len)()
    n = I32(-5)
    stops = (I32 * 17)(*range(17))
    cb = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.POINTER(I32), I32)()
    sp = len(PROMPT)
    bad = [
        (first, sp, 8, stops, 17, out, ctypes.byref(n)),  # n_stop > KLLM_MAX_STOP_IDS
        (first, sp, 8, stops, -1, out, ctypes.byref(n)),  # n_stop < 0
        (first, sp, 8, (I32 * 1)(shape.vocab_size), 1, out, ctypes.byref(n)),  # stop id >= vocab
        (first, sp, 8, (I32 * 1)(-1), 1, out, ctypes.byref(n)),  # stop id < 0
        (first, sp, shape.seq_len - sp + 1, stops, 1, out, ctypes.byref(n)),  # start_pos + max_steps > seq_len
        (first, sp, 0, stops, 1, out, ctypes.byref(n)),  # max_steps <= 0
        (first, sp, -3, stops, 1, out, ctypes.byref(n)),
        (first, sp, 8, stops, 1, None, ctypes.byref(n)),  # null out_tokens_host
        (first, sp, 8, stops, 1, out, None),  # null n_out
        (first, sp, 8, None, 2, out, ctypes.byref(n)),  # n_stop > 0 with null stop_ids
        (first, -1, 8, stops, 1, out, ctypes.byref(n)),
    ]
    for args in bad:
        f, p, m, s, ns, o, no = args
        assert lib.kllm_decoder_generate_until(dut.handle, f, p, m, s, ns, cb, None, o, no) == -1, args
    assert lib.kllm_decoder_generate_until(None, first, sp, 8, stops, 1, cb, None, out, ctypes.byref(n)) == -1
    k1, v1 = dut.kv_cache()
    assert_bit_equal(k1, k0, "kv after refusals")
    assert_bit_equal(v1, v0, "kv after refusals")
    assert_bit_equal(dut.logits(), lg0, "logits after refusals")
    # null stop_ids with n_stop == 0 and no callback is a valid call
    assert lib.kllm_decoder_generate_until(dut.handle, first, sp, 4, None, 0, cb, None, out, ctypes.byref(n)) == 0
    assert n.value == 4


def test_full_size_tinyllama_streams_while_it_runs(monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", "persistent")
    shape = SHAPES["tinyllama-1.1b"]
    w = synth_weights(shape, "cuda", 7)
    dut, ref = Decoder(shape, w), Decoder(shape, w)
    assert dut.engine == "persistent"
    M = 256
    full = ref.generate(1, 0, M)
    full_logits = ref.logits()
    dut.generate_until(1, 0, 8)  # warm-up
    calls = []
    t0 = time.perf_counter()
    ids = dut.generate_until(1, 0, M, on_tokens=lambda t: calls.append((time.perf_counter(), list(t))))
    wall = time.perf_counter() - t0
    assert ids == full
    assert [i for _, t in calls for i in t] == ids
    assert len(calls) > 1
    assert calls[0][0] - t0 < wall / 10, (calls[0][0] - t0, wall)
    assert_bit_equal(dut.logits(), full_logits, "tinyllama logits, no stop")
    for a, b in zip(kv_rows(dut, M), kv_rows(ref, M)):
        assert_bit_equal(a, b, "tinyllama kv, no stop")
    j = first_hits(full)[len(first_hits(full)) // 2]
    assert until(dut, 1, 0, M, [full[j]]) == full[:j + 1]
    ref.generate(1, 0, j + 1)
    assert_bit_equal(dut.logits(), ref.logits(), "tinyllama logits after a stop")
    assert dut.generate(full[j], j + 1, M - j - 1) == full[j + 1:]
    dut.close()
    ref.close()
