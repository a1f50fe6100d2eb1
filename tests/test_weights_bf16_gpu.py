"""-m gpu: bf16 weight matrices (kllm_decoder_desc::weights = KLLM_WEIGHTS_BF16).

The reference of every test is the fp32-weight decoder over the same weights rounded to bf16 and widened back to fp32
(decoder.bf16_weights, decoder.widen_weights).  Widening is exact and every operation stays fp32, so the bf16 decoder
must give the same bits: ids, logits and the kllm_decoder_read_kv cache.
  - every fp32 case of decode_model_util.CASES teacher-forced through its whole sequence: ids at every step, logits at
    the tile edges, the whole cache at the end; exact mode on both engines, fast mode on both engines at the same
    pinned ring geometry, and fast mode with the bf16 KV cache on the persistent engine;
  - fast mode at bf16's own default ring geometry within the fast-mode bounds of the fp64 model fed the widened
    weights;
  - every entry (prompt, generate, generate_until, sampling, penalties and bias, logprobs, score, prefill_tf32);
  - the op entries kllm_gemv_bf16 and kllm_gemm_bf16_tf32 against their fp32 forms;
  - TinyLlama-1.1B, Qwen2.5-0.5B and Llama-2-7B at full size;
  - the refusals, and the graph engine taking a shape the persistent ring does not.
"""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import (CASES, GEOMETRIES, KNOBS, WEIGHTS, case_id, device_sincos, edge_ends, engine_geometry,
                               run, same_bits, sequence, sms, taus)
from gpu_util import ptr, sync
from prefill_model import prefill_ref

from kuiperllama_b200 import ALLREDUCE_FN, SHAPES, Decoder, DecoderDesc, KllmError, synth_weights
from kuiperllama_b200.decoder import bf16_weights, widen_weights

pytestmark = pytest.mark.gpu

FP32_CASES = [c for c in CASES if GEOMETRIES[c[0]].group_size == 0]


def make(monkeypatch, shape, w, fmt, numerics="exact", engine=None, env=None, kv_cache="fp32"):
    for name in KNOBS:
        monkeypatch.delenv(name, raising=False)
    if engine is not None:
        monkeypatch.setenv("KLLM_ENGINE", engine)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    d = Decoder(shape, w, numerics=numerics, kv_cache=kv_cache, weight_format=fmt)
    if engine is not None:
        assert d.engine == engine
    return d


def pair(shape, seed=77, weights="synth"):
    w16 = bf16_weights(WEIGHTS[weights](shape, "cuda", seed))
    return w16, widen_weights(w16)


def assert_same_state(a, b, what):
    assert same_bits(a.logits(), b.logits()), (what, "logits")
    ka, va = a.kv_cache()
    kb, vb = b.kv_cache()
    assert same_bits(ka, kb) and same_bits(va, vb), (what, "kv cache")


def teacher_forced(dec, toks, ends):
    ids, logits, start = [], {}, 0
    for end in ends:
        ids += dec.generate(0, start, end + 1 - start, teacher=toks[start:end + 1])
        logits[end] = dec.logits()
        start = end + 1
    return ids, logits, dec.kv_cache()


def configs(shape):
    """(label, numerics, engine, env, kv_cache): the fast ones pin the fp32 decoder's default ring geometry."""
    T, SP, _, stage = engine_geometry(shape, "fast", {}, sms())
    pin = {"KLLM_STAGE_BYTES": str(stage), "KLLM_ATTN_SPLIT": str(SP)}
    out = [("exact-persistent", "exact", "persistent", {}, "fp32"), ("exact-graph", "exact", "graph", {}, "fp32"),
           ("fast-persistent", "fast", "persistent", pin, "fp32"), ("fast-graph", "fast", "graph", {}, "fp32")]
    if shape.head_size % 32 == 0:
        out.append(("fast-persistent-kv16", "fast", "persistent", pin, "bf16"))
    return out, edge_ends(T, SP, shape.seq_len)


@pytest.mark.parametrize("key,weights,env", FP32_CASES, ids=[case_id(c) for c in FP32_CASES])
def test_bitwise_equal_to_the_fp32_decoder_over_the_widened_weights(monkeypatch, key, weights, env):
    shape = GEOMETRIES[key]
    w16, w32 = pair(shape, weights=weights)
    toks = sequence(shape.vocab_size, shape.seq_len, 5)
    cfgs, ends = configs(shape)
    ring_takes_it = shape.dim % 8 == 0 and shape.hidden_dim % 8 == 0
    for label, numerics, engine, env_, kv in cfgs:
        if engine == "persistent" and not ring_takes_it:
            with pytest.raises(KllmError, match="-2"):
                make(monkeypatch, shape, w16, "bf16", numerics, engine, env_, kv)
            continue
        ref = make(monkeypatch, shape, w32, "fp32", numerics, engine, env_, kv)
        got = make(monkeypatch, shape, w16, "bf16", numerics, engine, env_, kv)
        if engine == "persistent":
            assert got.attention_geometry == ref.attention_geometry, label
        a, b = teacher_forced(ref, toks, ends), teacher_forced(got, toks, ends)
        assert a[0] == b[0], (key, label, "ids")
        for end in ends:
            assert same_bits(a[1][end], b[1][end]), (key, label, "logits", end)
        assert same_bits(a[2][0], b[2][0]) and same_bits(a[2][1], b[2][1]), (key, label, "kv cache")
        print("[weights-bf16]", key, label, f"{shape.seq_len} steps bit-identical", flush=True)
        ref.close()
        got.close()
    del w16, w32
    torch.cuda.empty_cache()


BOUND_CASES = [("small", "loud"), ("hs128", "loud"), ("small-qwen", "loud"), ("tinyllama-1.1b", "synth")]


@pytest.mark.parametrize("key,weights", BOUND_CASES, ids=[f"{k}-{w}" for k, w in BOUND_CASES])
def test_fast_mode_at_its_own_geometry_within_the_model_bounds(kllm_lib, monkeypatch, key, weights):
    shape = GEOMETRIES[key]
    w16, w32 = pair(shape, weights=weights)
    dec = make(monkeypatch, shape, w16, "bf16", "fast")
    assert dec.engine == "persistent"
    T, SP, _, stage = dec.attention_geometry
    ends = edge_ends(T, SP, shape.seq_len)
    toks = sequence(shape.vocab_size, shape.seq_len, 5)
    sin, cos = device_sincos(kllm_lib, shape)
    model = prefill_ref(w32, shape, toks, 0, sin, cos, tf32=False, logits_at=ends)
    kv_tau, logit_tau = taus(key)
    run(f"{key}-{weights} bf16 weights, stage {stage}", dec, shape, toks, model, ends, kv_tau, logit_tau,
        tag="[weights-bf16]")
    dec.close()


# ---- entries ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=["small", "small-qwen"])
def entry_pair(request):
    shape = replace(SHAPES[request.param], seq_len=320)
    w16, w32 = pair(shape, seed=2024)
    return shape, w16, w32


@pytest.mark.parametrize("engine", ["persistent", "graph"])
def test_every_entry_matches_the_fp32_decoder(monkeypatch, entry_pair, engine):
    shape, w16, w32 = entry_pair
    ref = make(monkeypatch, shape, w32, "fp32", engine=engine)
    got = make(monkeypatch, shape, w16, "bf16", engine=engine)
    V = shape.vocab_size
    prompt = [int(t) for t in np.random.default_rng(1).integers(0, V, 40)]

    def both(what, fn):
        ra, rb = fn(ref), fn(got)
        if isinstance(ra, np.ndarray):
            assert same_bits(ra, rb), (engine, what)
        elif isinstance(ra, tuple):
            for x, y in zip(ra, rb):
                assert same_bits(x, y) if isinstance(x, np.ndarray) else x == y, (engine, what)
        else:
            assert ra == rb, (engine, what)
        assert_same_state(ref, got, f"{engine} {what}")
        return ra

    nxt = both("prompt", lambda d: d.prompt(prompt))
    both("generate", lambda d: d.generate(nxt, len(prompt), 24))
    streamed = {id(ref): [], id(got): []}
    ids = ref.generate(nxt, len(prompt), 24)
    stops = [ids[17], ids[20]]
    both("generate_until", lambda d: (d.generate_until(nxt, len(prompt), 60, stops,
                                                       on_tokens=streamed[id(d)].extend), list(streamed[id(d)])))
    assert streamed[id(ref)] == streamed[id(got)] and 0 < len(streamed[id(ref)]) <= 18

    def sampled(d):
        d.set_sampling(0.9, 40, 7, top_p=0.85)
        out = d.generate(nxt, len(prompt), 32)
        d.set_sampling(0.0)
        return out
    both("sampling", sampled)

    def penalised(d):
        d.set_repetition_penalty(1.3, 16)
        d.set_frequency_presence(0.4, 0.2, len(prompt))
        d.set_logit_bias({3: 2.5, 11: -100.0})
        out = d.generate(nxt, len(prompt), 32)
        d.set_repetition_penalty(1.0)
        d.set_frequency_presence(0.0, 0.0)
        d.set_logit_bias()
        return out
    both("penalties", penalised)

    def logprobs(d):
        d.set_logprobs(5)
        out = d.generate(nxt, len(prompt), 16)
        rec = d.logprobs(len(prompt), 16)
        d.set_logprobs(-1)
        return (out,) + rec
    both("logprobs", logprobs)
    both("score", lambda d: d.score(prompt + ids[:20]))
    both("prefill_tf32", lambda d: d.prefill_tf32(prompt[:37], 3))
    both("step after prefill", lambda d: d.step(prompt[37], 40))
    ref.close()
    got.close()


# ---- op entries ------------------------------------------------------------------------------------------------------
GEMV_SHAPES = [(1, 1), (3, 5), (4, 7), (127, 33), (128, 129), (512, 130), (513, 257), (2048, 1000), (5632, 96)]


@pytest.mark.parametrize("in_dim,out_dim", GEMV_SHAPES)
@pytest.mark.parametrize("offset", [0, 1])
def test_gemv_bf16_matches_gemv_f32(kllm_lib, in_dim, out_dim, offset):
    g = torch.Generator(device="cuda").manual_seed(in_dim * 7 + out_dim)
    x = torch.randn(in_dim, device="cuda", generator=g)
    base = torch.randn(out_dim * in_dim + offset, device="cuda", generator=g).to(torch.bfloat16)
    w16 = base[offset:]  # offset 1: rows off the 8-byte alignment of the vector loads
    w32 = w16.float().contiguous()
    a = torch.empty(out_dim, device="cuda")
    b = torch.empty(out_dim, device="cuda")
    assert kllm_lib.kllm_gemv_f32(ptr(x), ptr(w32), ptr(a), in_dim, out_dim, None) == 0
    assert kllm_lib.kllm_gemv_bf16(ptr(x), ptr(w16), ptr(b), in_dim, out_dim, None) == 0
    sync()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("n_tokens", [1, 255, 256, 257])
@pytest.mark.parametrize("in_dim,out_dim", [(512, 200), (1032, 384)])
def test_gemm_bf16_tf32_matches_gemm_tf32(kllm_lib, n_tokens, in_dim, out_dim):
    g = torch.Generator(device="cuda").manual_seed(n_tokens + in_dim)
    x = torch.randn(n_tokens, in_dim, device="cuda", generator=g)
    w16 = torch.randn(out_dim, in_dim, device="cuda", generator=g).to(torch.bfloat16)
    w32 = w16.float().contiguous()
    a = torch.empty(n_tokens, out_dim, device="cuda")
    b = torch.full((n_tokens, out_dim), float("nan"), device="cuda")
    assert kllm_lib.kllm_gemm_tf32(ptr(x), ptr(w32), ptr(a), n_tokens, in_dim, out_dim, None) == 0
    assert kllm_lib.kllm_gemm_bf16_tf32(ptr(x), ptr(w16), ptr(b), n_tokens, in_dim, out_dim, None) == 0
    sync()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert kllm_lib.kllm_gemm_bf16_tf32(ptr(x), ptr(w16), ptr(b), n_tokens, 516, out_dim, None) == -2  # in_dim % 8


# ---- full-size shapes ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tinyllama-1.1b", "qwen2.5-0.5b", "llama2-7b"])
def test_full_size_models(monkeypatch, name):
    shape = replace(SHAPES[name], seq_len=256)
    w32 = synth_weights(shape, "cuda", 1238)
    w16 = bf16_weights(w32)
    del w32
    torch.cuda.empty_cache()
    wide = widen_weights(w16)
    free, total = torch.cuda.mem_get_info()
    for numerics in ("exact", "fast"):
        ref = make(monkeypatch, shape, wide, "fp32", numerics)
        got = make(monkeypatch, shape, w16, "bf16", numerics, env={"KLLM_STAGE_BYTES": str(
            ref.attention_geometry[3])})
        assert got.engine == ref.engine == "persistent"
        prompt = [1, 2, 3, 5, 8, 13, 21, 34]
        a, b = ref.prompt(prompt), got.prompt(prompt)
        assert a == b
        assert ref.generate(a, len(prompt), 40) == got.generate(b, len(prompt), 40), (name, numerics)
        assert_same_state(ref, got, f"{name} {numerics}")
        ref.close()
        got.close()
    mat = sum(w16[n].numel() for n in ("wq", "wk", "wv", "wo", "w1", "w2", "w3", "wcls"))
    print("[weights-bf16]", name, f"40 steps bit-identical in both modes; matrices {mat * 2 / 1e9:.2f} GB in bf16 "
          f"against {mat * 4 / 1e9:.2f} GB in fp32 (free {free / 1e9:.1f} of {total / 1e9:.1f} GB)", flush=True)
    del w16, wide
    torch.cuda.empty_cache()


# ---- refusals and the graph engine -----------------------------------------------------------------------------------
def test_refusals_create_nothing(kllm_lib, monkeypatch):
    shape = replace(SHAPES["small"], seq_len=64)
    w16, _ = pair(shape, seed=3)
    for name in KNOBS:
        monkeypatch.delenv(name, raising=False)
    dec = Decoder(shape, w16, weight_format="bf16")

    def create(**fields):
        d = DecoderDesc.from_buffer_copy(dec.desc)
        for k, v in fields.items():
            setattr(d, k, v)
        h = ctypes.c_void_p()
        rc = kllm_lib.kllm_decoder_create(ctypes.byref(d), None, ctypes.byref(h))
        assert not h.value, fields  # nothing created
        return rc

    assert create(weights=2) == -1
    assert create(weights=-1) == -1
    assert create(group_size=64) == -1
    cb = ALLREDUCE_FN(lambda ctx, buf, n, s: 0)
    assert create(tp_size=3, tp_rank=0, allreduce=cb, dim=shape.dim, head_num=shape.head_num // 3,
                  kv_head_num=shape.kv_head_num // 3) == -2
    n = ctypes.c_int32(-1)
    toks = (ctypes.c_int32 * 4)(1, 2, 3, 4)
    assert kllm_lib.kllm_decoder_prefill_w8(dec.handle, toks, 4, 0, ctypes.byref(n)) == -2
    stamps = (ctypes.c_uint64 * 4096)()
    g, p = ctypes.c_int32(0), ctypes.c_int32(0)
    assert kllm_lib.kllm_decoder_profile(dec.handle, 1, 0, 2, 0, stamps, 4096, ctypes.byref(g), ctypes.byref(p)) == -2
    with pytest.raises(KllmError):  # the Python side refuses fp32 tensors under weight_format="bf16"
        Decoder(shape, widen_weights(w16), weight_format="bf16")
    dec.close()


def test_hs16_runs_on_the_graph_engine(monkeypatch):
    shape = replace(GEOMETRIES["hs16"], seq_len=64)
    w16, w32 = pair(shape, weights="loud")
    got = make(monkeypatch, shape, w16, "bf16")
    assert got.engine == "graph"
    ref = make(monkeypatch, shape, w32, "fp32", engine="graph")
    assert ref.generate(1, 0, 40) == got.generate(1, 0, 40)
    assert_same_state(ref, got, "hs16")
    with pytest.raises(KllmError, match="-2"):
        make(monkeypatch, shape, w16, "bf16", engine="persistent")
    ref.close()
    got.close()


# ---- the long-row chunks, every step's logits, the refused prefill ------------------------------------------------
def test_long_rows_split_into_chunks(monkeypatch):
    """2 KB ring stages: W2's 1536-wide rows (3 KB in bf16) span two stages, the fp32 rows three -- the long-row path of
    both row accumulators -- while the SwiGLU pairs of 256-wide rows still fit.  Bitwise, every step."""
    from kuiperllama_b200 import ModelShape
    shape = ModelShape("chunk-rows", 256, 1536, 2, 16, 4, 512, 256)
    w16, w32 = pair(shape, weights="loud")
    toks = sequence(shape.vocab_size, shape.seq_len, 5)
    env = {"KLLM_STAGE_BYTES": "2048"}
    for numerics in ("exact", "fast"):
        ref = make(monkeypatch, shape, w32, "fp32", numerics, "persistent", env)
        got = make(monkeypatch, shape, w16, "bf16", numerics, "persistent", env)
        assert got.attention_geometry == ref.attention_geometry and got.attention_geometry[3] == 2048
        ends = list(range(shape.seq_len))
        a, b = teacher_forced(ref, toks, ends), teacher_forced(got, toks, ends)
        assert a[0] == b[0], numerics
        for end in ends:
            assert same_bits(a[1][end], b[1][end]), (numerics, end)
        assert same_bits(a[2][0], b[2][0]) and same_bits(a[2][1], b[2][1]), numerics
        ref.close()
        got.close()


@pytest.mark.parametrize("engine", ["persistent", "graph"])
@pytest.mark.parametrize("numerics", ["exact", "fast"])
def test_logits_bitwise_at_every_step(monkeypatch, engine, numerics):
    """Teacher-forced one position per call over a whole sequence: the logits of every step, then the cache."""
    shape = replace(GEOMETRIES["small-qwen"], seq_len=288)
    w16, w32 = pair(shape, weights="loud")
    toks = sequence(shape.vocab_size, shape.seq_len, 5)
    env = {}
    if engine == "persistent" and numerics == "fast":
        _, SP, _, stage = engine_geometry(shape, "fast", {}, sms())
        env = {"KLLM_STAGE_BYTES": str(stage), "KLLM_ATTN_SPLIT": str(SP)}
    ref = make(monkeypatch, shape, w32, "fp32", numerics, engine, env)
    got = make(monkeypatch, shape, w16, "bf16", numerics, engine, env)
    a, b = teacher_forced(ref, toks, list(range(shape.seq_len))), teacher_forced(got, toks, list(range(shape.seq_len)))
    assert a[0] == b[0]
    for pos in range(shape.seq_len):
        assert same_bits(a[1][pos], b[1][pos]), pos
    assert same_bits(a[2][0], b[2][0]) and same_bits(a[2][1], b[2][1])
    ref.close()
    got.close()


def test_refused_prefill_leaves_the_decoder_as_it_was(monkeypatch):
    """hs16's hidden rows (172) are not a multiple of 8, which kllm_gemm_bf16_tf32 needs: prefill_tf32 is refused
    before any launch, and logits, cache and history stay as the decoder had them."""
    shape = replace(GEOMETRIES["hs16"], seq_len=64)
    w16, _ = pair(shape, weights="loud")
    dec = make(monkeypatch, shape, w16, "bf16")
    dec.generate(1, 0, 12)
    before = (dec.logits(), *dec.kv_cache(), dec.history())
    with pytest.raises(KllmError, match="-2"):
        dec.prefill_tf32([3, 4, 5, 6, 7], 2)
    after = (dec.logits(), *dec.kv_cache(), dec.history())
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
    dec.close()
