"""-m gpu: the bf16 KV cache (kllm_decoder_desc::kv_cache = KLLM_KV_BF16) of the fast decode mode.

Against the fp64 model (tests/kv_bf16_model.py, rule "decode"), teacher-forced over every position of the decode-model
cases whose head size the bf16 tile mapping takes (head_size % 32 == 0), and of bf16 weights at their own ring stage
(the model fed the weights widened to fp32), at the flash geometry's tile and split edges.
The model is fed the GPU's own cache rows (kv_rows): each position attends over the rows the decoder cached, which
isolates the kernel from the rounding -- a row whose fp32 value lies on the other side of a rounding boundary on the
GPU than in the model differs by one ulp, and with sharp attention that moves every later row of the next layers by
far more than the fp32 bound.  Then:
  - every read_kv element is a bf16 value within one bf16 ulp plus KV_TAU * rms(row) of the model's rounded row;
  - the logits are within the fast-mode bound (LOGIT_TAU * rms) of the model;
  - and within BF16_GAIN x the bf16 model's own distance from the fp32-cache model, plus that bound, of the
    fp32-cache model: the kernel's distance from the fp32 model is at most its distance from the bf16 model plus the
    bf16 model's from the fp32 one (triangle inequality); the factor covers the rows where the GPU's fp32 value lies
    on the other side of a bf16 rounding boundary than the model's (one ulp).
Entries: prompt, generate and generate_until equal stepping bit for bit; sampled and penalised ids follow the rule of
kuiperllama_b200/sampling.py on the bf16 decoder's logits; both batched prefills write bf16 rows within their bounds,
and decode continues from them across a tile edge within the fast-mode bound of the model; Llama-2-7B int8 at seq_len
4096 decoding past position 4000 agrees
with the fp32 cache; the cache takes half the memory; every refusal of kllm_decoder_create.

Measured worst values (an NVIDIA H100 80GB HBM3 at a 700 W power limit) are printed with the [kv-bf16] tag.
"""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import (CASES, GEOMETRIES, KNOBS, LOGIT_TAU, WEIGHTS, case_id, continue_ends, device_sincos,
                               engine_geometry, sequence, sms, taus)
from kv_bf16_model import bf16_rne, prefill_ref_bf16
from prefill_model import prefill_ref

from kuiperllama_b200 import ALLREDUCE_FN, SHAPES, Decoder, KllmError, synth_weights
from kuiperllama_b200 import sampling as ref_sampling
from kuiperllama_b200.decoder import bf16_weights, widen_weights

pytestmark = pytest.mark.gpu

# Measured worst values, an NVIDIA H100 80GB HBM3 at 700 W: K / V err / (ulp + KV_TAU rms) 0.999 (tinyllama-1.1b);
# logits err / fast-mode bound against the model on the GPU's rows 0.228 (tinyllama-1.1b); distance from the fp32-cache
# model over the bf16 model's own distance 1.01 (small-loud, KLLM_ATTN_SPLIT=2), against BF16_GAIN.  bf16 weights at
# their own 24 KB stage (same card and limit): K / V 0.997 (hs128), logits 0.0931 (gqa-hs64, KLLM_ATTN_SPLIT=4),
# distance 1.00 of the bf16 model's own (hs128).  Decode after the batched prefill, logits err / fast-mode bound:
# 0.0244 (small-int8), 0.014 (small).
BF16_GAIN = 2.0
# (geometry, weights, environment, weight format)
BF16_CASES = [c + ("int8" if GEOMETRIES[c[0]].group_size else "fp32",) for c in CASES
              if GEOMETRIES[c[0]].head_size % 32 == 0]
# tile and split geometries of the bf16 cache: a smaller ring stage and a smaller split on one case each
BF16_CASES += [("hs128", "loud", {"KLLM_STAGE_BYTES": "8192"}, "fp32"),
               ("small", "loud", {"KLLM_ATTN_SPLIT": "2"}, "fp32"),
               ("llama2-7b-int8-2l", "outliers", {"KLLM_STAGE_BYTES": "16384", "KLLM_ATTN_SPLIT": "2"}, "int8")]
# bf16 weights at their 24 KB stages: T = 96 at hs 128, T = 192 at hs 64 (a split of 4 puts SP * T inside the sequence)
BF16_CASES += [("hs128", "loud", {}, "bf16"), ("gqa-hs64", "loud", {}, "bf16"),
               ("gqa-hs64", "loud", {"KLLM_ATTN_SPLIT": "4"}, "bf16")]


def report(*parts):
    print("[kv-bf16]", *parts, flush=True)


def bf16_id(c):
    return case_id(c[:3]) + ("-bf16w" if c[3] == "bf16" else "")


def make(monkeypatch, shape, w, env=None, kv_cache="bf16", numerics="fast", weight_format="fp32"):
    for name in KNOBS:
        monkeypatch.delenv(name, raising=False)
    for name, value in (env or {}).items():
        monkeypatch.setenv(name, value)
    return Decoder(shape, w, numerics=numerics, kv_cache=kv_cache, weight_format=weight_format)


def bf16_geometry(shape, env, weight_format="fp32"):
    """(T, SP) of the flash form with a bf16 cache (decode_model_util.engine_geometry): the weight format's stage,
    T = min(stage / (hs * 2), 256) & ~31, the split as fp32's."""
    return engine_geometry(shape, "fast", env, sms(), "bf16", weight_format)[:2]


def ends_for(T, SP, seq_len):
    e = {0, 1, 7, 8, 9, T - 1, T, T + 1, SP * T - 1, SP * T, SP * T + 1, seq_len - 1}
    return sorted(p for p in e if 0 <= p < seq_len)


def ulp_bf16(x):
    """One bf16 ulp at |x| (the spacing of bf16 values at that magnitude; 2^-133 for subnormals and zero)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


@pytest.mark.parametrize("key,weights,env,weight_format", BF16_CASES, ids=[bf16_id(c) for c in BF16_CASES])
def test_bf16_decode_against_the_model(kllm_lib, monkeypatch, key, weights, env, weight_format):
    shape = GEOMETRIES[key]
    w = WEIGHTS[weights](shape, "cuda", 77)
    w_dec = bf16_weights(w) if weight_format == "bf16" else None
    decode_against_the_bf16_model(kllm_lib, monkeypatch, bf16_id((key, weights, env, weight_format)), shape,
                                  w if w_dec is None else widen_weights(w_dec), env, *taus(key), w_dec=w_dec)


def decode_against_the_bf16_model(kllm_lib, monkeypatch, what, shape, w, env, kv_tau, logit_tau, tag="[kv-bf16]",
                                  w_dec=None):
    """One bf16-cache decoder teacher-forced over every position in segments ending on the edges of the tiles it
    reports (which must be bf16_geometry's), held to the bounds of the module docstring.  w_dec: bf16 weights for the
    decoder (decoder.bf16_weights), w then being their widening; None runs the decoder over w."""
    weight_format = "fp32" if w_dec is None else "bf16"
    T, SP = bf16_geometry(shape, env, weight_format)
    ends = ends_for(T, SP, shape.seq_len)
    toks = sequence(shape.vocab_size, shape.seq_len, 5)
    sin, cos = device_sincos(kllm_lib, shape)
    fixed = shape.group_size == 64
    model = prefill_ref_bf16(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends, fixed_point=fixed,
                             rule="decode")
    plain = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends, fixed_point=fixed)
    dec = make(monkeypatch, shape, w if w_dec is None else w_dec, env, weight_format=weight_format)
    assert dec.engine == "persistent"
    assert dec.attention_geometry == engine_geometry(shape, "fast", env, sms(), "bf16", weight_format), \
        (what, dec.attention_geometry)
    start, logits = 0, {}
    for end in ends:
        dec.generate(0, start, end + 1 - start, teacher=toks[start:end + 1])
        logits[end] = torch.from_numpy(dec.logits()).cuda().double()
        start = end + 1
    k, v = (torch.from_numpy(a).cuda() for a in dec.kv_cache())
    fed = prefill_ref_bf16(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends, fixed_point=fixed, rule="decode",
                           kv_rows=(k, v))
    # (1) the cache: bf16 values, within one ulp + KV_TAU * rms of the model's rounded rows
    worst_kv = 0.0
    for name, got, ref in (("K", k, fed["k"]), ("V", v, fed["v"])):
        assert torch.equal(bf16_rne(got), got.float()), f"{name}: a cached element is not a bf16 value"
        want = bf16_rne(ref).double()
        rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
        bound = ulp_bf16(want) + kv_tau * rms
        r = float(((got.double() - want).abs() / bound).max())
        worst_kv = max(worst_kv, r)
        assert r <= 1.0, (what, name, r)
    # (2) the logits against the model fed the GPU's own cache rows, (3) against the fp32-cache model
    worst_own, worst_plain, rule_dist = 0.0, 0.0, 0.0
    for end in ends:
        own = fed["logits_at"][end]
        rms = float(own.pow(2).mean().sqrt())
        worst_own = max(worst_own, float((logits[end] - own).abs().max()) / (logit_tau * rms))
        rule_dist = max(rule_dist, float((model["logits_at"][end] - plain["logits_at"][end]).abs().max()) / rms)
        worst_plain = max(worst_plain, float((logits[end] - plain["logits_at"][end]).abs().max()) / rms)
    plain_bound = BF16_GAIN * rule_dist + logit_tau
    print(tag, f"{what} T={T} SP={SP}: K/V err / (ulp + tau rms) {worst_kv:.3g}; logits err / "
          f"fast bound vs model on GPU rows {worst_own:.3g}; vs fp32-cache model err / rms {worst_plain:.3g} "
          f"(bound {plain_bound:.3g}, bf16 model's own distance {rule_dist:.3g})", flush=True)
    assert worst_own <= 1.0, (what, worst_own)
    assert worst_plain <= plain_bound, (what, worst_plain, plain_bound)
    dec.close()


# ---- entries ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small():
    shape = replace(SHAPES["small-int8"], seq_len=640)
    return shape, synth_weights(shape, "cuda", 2024)


def same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def test_entries_match_stepping(kllm_lib, monkeypatch, small):
    shape, w = small
    toks = sequence(shape.vocab_size, 300, 9)
    a, b = make(monkeypatch, shape, w), make(monkeypatch, shape, w)
    for p, t in enumerate(toks[:-1]):
        a.step(t, p, is_prompt=True)
    nxt = a.step(toks[-1], len(toks) - 1)
    assert b.prompt(toks) == nxt and same(a.logits(), b.logits())
    ka, va = a.kv_cache()
    kb, vb = b.kv_cache()
    assert same(ka, kb) and same(va, vb)
    ids_step, tok = [], nxt
    for p in range(len(toks), len(toks) + 40):
        tok = a.step(tok, p)
        ids_step.append(tok)
    ids_gen = b.generate(nxt, len(toks), 40)
    assert list(ids_gen) == ids_step and same(a.logits(), b.logits())
    d = make(monkeypatch, shape, w)
    d.prompt(toks)
    assert d.generate_until(nxt, len(toks), 40) == ids_step and same(d.logits(), b.logits())
    kd, vd = d.kv_cache()
    ka, va = a.kv_cache()
    assert same(ka, kd) and same(va, vd)
    for x in (a, b, d):
        x.close()


def test_sampling_and_penalties_follow_the_rule(kllm_lib, monkeypatch, small):
    shape, w = small
    toks = sequence(shape.vocab_size, 64, 3)
    dec = make(monkeypatch, shape, w)
    temperature, top_k, seed, top_p, penalty, freq, pres = 0.8, 40, 7, 0.9, 1.3, 0.4, 0.2
    dec.set_sampling(temperature, top_k, seed, top_p)
    dec.set_repetition_penalty(penalty, 0)
    dec.set_frequency_presence(freq, pres, 0)
    nxt = dec.prompt(toks)
    hist, tok, checked = list(toks), nxt, 0
    for p in range(len(toks), len(toks) + 48):
        hist.append(tok)
        tok = dec.step(tok, p)
        logits = dec.logits()
        adj = ref_sampling.penalties(logits, rep_ids=np.array(hist), penalty=penalty, count_ids=np.array(hist),
                                     frequency=freq, presence=pres)
        if ref_sampling.margin(adj, temperature, top_k, seed, p, top_p) > 1e-5:
            assert tok == ref_sampling.sample(adj, temperature, top_k, seed, p, top_p), p
            checked += 1
    report(f"sampled ids checked against the rule: {checked} of 48")
    assert checked >= 40
    dec.close()


@pytest.mark.parametrize("key", ["small", "small-int8"])
def test_batched_prefill_writes_bf16_rows_and_decode_continues(kllm_lib, monkeypatch, key):
    shape = replace(SHAPES[key], seq_len=640)
    w = synth_weights(shape, "cuda", 31)
    toks = sequence(shape.vocab_size, 400, 6)
    sin, cos = device_sincos(kllm_lib, shape)
    dec = make(monkeypatch, shape, w)
    nxt = dec.prefill_w8(toks) if shape.group_size else dec.prefill_tf32(toks)
    k, v = (torch.from_numpy(a).cuda() for a in dec.kv_cache())
    model = prefill_ref_bf16(w, shape, toks, 0, sin, cos, tf32=True, rule="prefill")
    n = len(toks)
    tau = 5e-2 if shape.group_size else 1e-2  # the prefill bounds (include/kllm_b200.h, tests/test_prefill_*.py)
    worst = 0.0
    for name, got, ref in (("K", k[:, :n], model["k"]), ("V", v[:, :n], model["v"])):
        assert torch.equal(bf16_rne(got), got.float()), name
        want = bf16_rne(ref).double()
        bound = ulp_bf16(want) + tau * (ref.pow(2).mean(-1, keepdim=True).sqrt() + 1e-3)
        worst = max(worst, float(((got.double() - want).abs() / bound).max()))
    report(f"{key} prefill rows err / (ulp + prefill bound) {worst:.3g}")
    assert worst <= 1.0
    lg = torch.from_numpy(dec.logits()).cuda().double()
    assert float((lg - model["logits"]).abs().max()) <= 2e-2 * float(model["logits"].abs().max())
    # decode continues over the prefilled bf16 rows, teacher-forced across the next tile edge: each segment end's logits
    # within the fast-mode bound of the model attending over the GPU's prefilled rows (kv_in) and decoded rows (kv_rows)
    assert dec.attention_geometry == engine_geometry(shape, "fast", {}, sms(), "bf16"), dec.attention_geometry
    ends = continue_ends(dec.attention_geometry[0], n, shape.seq_len)
    more = sequence(shape.vocab_size, ends[-1] + 1 - n, 16)
    start, logits = n, {}
    for end in ends:
        dec.generate(0, start, end + 1 - start, teacher=more[start - n:end + 1 - n])
        logits[end] = torch.from_numpy(dec.logits()).cuda().double()
        start = end + 1
    k, v = (torch.from_numpy(a).cuda() for a in dec.kv_cache())
    fed = prefill_ref_bf16(w, shape, more, n, sin, cos, tf32=False, logits_at=[e - n for e in ends],
                           fixed_point=shape.group_size == 64, rule="decode", kv_in=(k, v),
                           kv_rows=(k[:, n:], v[:, n:]))
    worst = max(float((logits[e] - fed["logits_at"][e - n]).abs().max())
                / (LOGIT_TAU * float(fed["logits_at"][e - n].pow(2).mean().sqrt())) for e in ends)
    report(f"{key} decode after the prefill, segments {ends}: logits err / fast bound {worst:.3g}")
    assert worst <= 1.0
    dec.close()


def test_long_context_llama2_7b_int8_agrees_with_the_fp32_cache(kllm_lib, monkeypatch):
    """Llama-2-7B int8 at seq_len 4096: both caches filled by the batched prefill to position 4000, then 60 decode
    steps teacher-forced; logits within 2e-2 * max|logit| of the fp32 cache's (the int8 prefill's bound), greedy ids
    equal wherever the fp32 cache's top-2 margin exceeds twice that."""
    shape = replace(SHAPES["llama2-7b-int8"], seq_len=4096)
    w = synth_weights(shape, "cuda", 1234)
    toks = sequence(shape.vocab_size, 4060, 12)
    worst = 0.0
    decs = [make(monkeypatch, shape, w, kv_cache=c) for c in ("fp32", "bf16")]
    for d in decs:
        d.prefill_w8(toks[:4000])
    for p in range(4000, 4060, 6):
        out = []
        for d in decs:
            d.generate(0, p, 6, teacher=toks[p:p + 6])
            out.append(d.logits())
        a, b = out
        bound = 2e-2 * float(np.abs(a).max())
        worst = max(worst, float(np.abs(a - b).max()) / bound)
        top2 = np.sort(a)[-2:]
        if top2[1] - top2[0] > 2 * bound:
            assert int(np.argmax(a)) == int(np.argmax(b)), p
    report(f"Llama-2-7B int8 pos 4000..4059: |bf16 - fp32 cache| / (2e-2 max|logit|) {worst:.3g}")
    assert worst <= 1.0
    for d in decs:
        d.close()


def test_cache_memory_is_halved(kllm_lib, monkeypatch):
    shape = replace(SHAPES["llama2-7b-int8"], layer_num=4, seq_len=4096)
    w = synth_weights(shape, "cuda", 5)
    used = {}
    for c in ("fp32", "bf16"):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        d = make(monkeypatch, shape, w, kv_cache=c)
        used[c] = free0 - torch.cuda.mem_get_info()[0]
        d.close()
    kv = 2 * shape.layer_num * shape.seq_len * shape.kv_dim * 4  # K and V, fp32 bytes
    report(f"create's allocation: fp32 cache {used['fp32'] / 2**20:.1f} MiB, bf16 {used['bf16'] / 2**20:.1f} MiB; "
           f"fp32 K+V {kv / 2**20:.1f} MiB")
    assert abs((used["fp32"] - used["bf16"]) - kv / 2) <= 8 * 2 ** 20


# ---- refusals --------------------------------------------------------------------------------------------------------
def rc_of(fn):
    """The return code of kllm_decoder_create behind a Decoder(...) call, 0 when it succeeded."""
    try:
        fn().close()
    except KllmError as e:
        return int(str(e).split("failed: ")[1].split()[0])
    return 0


@pytest.mark.parametrize("what", ["exact", "mode-env-exact", "engine-graph", "tp2", "hs48", "hs16", "hs256"])
def test_refusals(kllm_lib, monkeypatch, what):
    shape, w, env, kw = SHAPES["small"], None, {}, {}
    if what == "exact":
        kw["numerics"] = "exact"
    elif what == "mode-env-exact":
        env["KLLM_MODE"] = "exact"
    elif what == "engine-graph":
        env["KLLM_ENGINE"] = "graph"
    elif what == "hs48":
        shape = SHAPES["small-hs48"]
    elif what == "hs16":
        shape = GEOMETRIES["hs16"]
    elif what == "hs256":  # head_size 256: the persistent engine's tiles stop at 128; only the graph engine runs it
        shape = replace(SHAPES["small"], name="hs256", dim=512, head_num=2, kv_head_num=2)
    w = synth_weights(shape, "cuda", 3)
    if what == "tp2":
        cb = ALLREDUCE_FN(lambda ctx, buf, n, s: 0)
        rc = rc_of(lambda: Decoder(shape, w, tp_size=2, tp_rank=0, allreduce=cb, numerics="fast", kv_cache="bf16"))
    else:
        rc = rc_of(lambda: make(monkeypatch, shape, w, env, **kw))
    assert rc == -2, (what, rc)
    # and the fp32 cache is not refused where it runs
    if what in ("exact", "mode-env-exact", "engine-graph", "hs48", "hs16"):
        make(monkeypatch, shape, w, env, kv_cache="fp32", numerics=kw.get("numerics", "fast")).close()


def test_unknown_kv_cache_value_is_invalid(kllm_lib, monkeypatch, small):
    shape, w = small
    d = make(monkeypatch, shape, w, kv_cache="fp32")
    desc = d.desc
    desc.kv_cache = 2
    h = ctypes.c_void_p()
    assert kllm_lib.kllm_decoder_create(ctypes.byref(desc), None, ctypes.byref(h)) == -1
    d.close()


# ---- C++ host: KUIPER_KV_CACHE=bf16 --------------------------------------------------------------------------------
def test_cpp_bf16_kv_cache_matches_the_cabi(kllm_lib, tmp_path, monkeypatch):
    import os
    from test_z_host_cpp import ensure_built, run_decode
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = SHAPES["small-int8"]
    w = synth_weights(shape, "cuda", 77)
    path = tmp_path / "small-int8.bin"
    write_checkpoint(str(path), shape, w)
    prompt, steps = [1, 5, 9], 60
    dec = make(monkeypatch, shape, w)
    want, tok = [], None
    for pos in range(steps):
        tok = dec.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
        want.append(tok)
    dec.close()
    want = want[len(prompt) - 1:]
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env["KUIPER_NUMERICS"] = "fast"
    r = run_decode("llama2", path, "llama", "int8", steps, prompt, env=dict(env, KUIPER_KV_CACHE="bf16"))
    assert r.returncode == 0, r.stderr
    assert [int(x) for x in r.stdout.split()][len(prompt) - 1:] == want
    cmd = [str(ensure_built("llama2")), str(path), "llama", "int8", str(steps), *map(str, prompt), "--kv-cache", "bf16"]
    import subprocess
    r2 = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env)
    assert r2.returncode == 0, r2.stderr
    assert r2.stdout.split() == r.stdout.split()
    # without the fast numerics init() fails rather than run an fp32 cache
    env.pop("KUIPER_NUMERICS")
    r3 = run_decode("llama2", path, "llama", "int8", steps, prompt, env=dict(env, KUIPER_KV_CACHE="bf16"))
    assert r3.returncode != 0 and "bf16" in r3.stderr
