"""-m gpu: the fp8 KV cache (kllm_decoder_desc::kv_cache = KLLM_KV_FP8) of the fast decode mode.

Against the fp64 model (tests/kv_fp8_model.py, rule "decode"), teacher-forced over every position of decode-model
geometries whose head size the fp8 tile mapping takes (head_size % 64 == 0), with fp32, int8 and bf16 weights (the
model fed bf16 weights widened to fp32, and the int8 decode step's fixed point), with unit scales and with scales
calibrated on the model's fp32 rows (decoder.fp8_kv_scales), at the flash geometry's tile and split edges and at
smaller stages and splits.  As in tests/test_kv_bf16_gpu.py the model is fed the GPU's own cache rows
(kv_rows), so each position attends over the rows the decoder cached.  Then:
  - every read_kv element is within one e4m3 ulp (at its magnitude, times its scale) plus KV_TAU * rms(row) of the
    model's rounded row, and where the model's scaled value lies farther than that tolerance from an e4m3 rounding
    boundary, it is exactly the model's code's value;
  - the logits are within the fast-mode bound (LOGIT_TAU * rms) of the model;
  - and within FP8_GAIN x the fp8 model's own distance from the fp32-cache model, plus that bound, of the fp32-cache
    model.
Entries: prompt, generate and generate_until equal stepping bit for bit; sampled and penalised ids follow
kuiperllama_b200/sampling.py on the decoder's logits; both batched prefills write fp8 rows, and decode continues from
them across a tile edge within the fast-mode bound of the model; bf16 weights over the fp8 cache equal fp32 weights
over the widened ones bit for bit; Llama-2-7B int8 at seq_len 4096 agrees with the fp32 cache past position 4000; the
cache takes a quarter of the memory; every refusal; the C++ host against the C ABI.

Measured worst values (an NVIDIA H100 80GB HBM3 at a 700 W power limit) are printed with the [kv-fp8] tag.  Of the
int8-weight cases: K / V err / (ulp + KV_TAU rms) 1.00 (llama2-7b-int8-2l, one ulp where the GPU's fp32 value and the
model's lie on either side of a rounding boundary), logits err / fast-mode bound 0.0575 (llama2-7b-int8-2l,
calibrated), distance from the fp32-cache model 1.00 of the fp8 model's own (FP8_GAIN 2).  Of the bf16-weight cases:
K / V 1.00 (hs128), logits 0.0659 (hs128, calibrated), distance 1.00 of the fp8 model's own.  Decode after the
batched prefill, logits err / fast-mode bound: 0.0233 (small-int8), 0.0102 (prefill-hs64).  These int8- and
bf16-weight cases, the bf16 cache's bf16-weight cases and the log-probability kernel pairs of test_logprobs_gpu.py
take about 7 s together on that card.
"""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import (GEOMETRIES, KNOBS, LOGIT_TAU, WEIGHTS, case_id, continue_ends, device_sincos,
                               engine_geometry, sequence, sms, taus)
from kv_fp8_model import e4m3_rne, fp8_round_rows, per_head, prefill_ref_fp8, ulp_e4m3
from prefill_model import prefill_ref

from kuiperllama_b200 import ALLREDUCE_FN, SHAPES, Decoder, KllmError, ModelShape, synth_weights
from kuiperllama_b200 import sampling as ref_sampling
from kuiperllama_b200.decoder import bf16_weights, fp8_kv_scales, widen_weights

pytestmark = pytest.mark.gpu

FP8_GAIN = 2.0
# Llama-2-7B int8 past position 4000: |fp8 - fp32 cache| / max|logit|, measured 0.175 (the bf16 cache: 0.013) on an
# NVIDIA H100 80GB HBM3 at 700 W
LONG_BOUND = 0.3
# (geometry, weights, environment, calibrated scales, weight format)
FP8_CASES = [(key, weights, env, calibrated, "fp32")
             for key, weights, env in [("hs128", "loud", {}), ("qwen2.5-reduced", "synth", {}),
                                       ("llama3-reduced", "loud", {}), ("gqa-hs64", "loud", {})]
             for calibrated in (False, True)]
# smaller stages and splits: T = 64 at hs128, and a split of 2
FP8_CASES += [("hs128", "loud", {"KLLM_STAGE_BYTES": "8192"}, True, "fp32"),
              ("gqa-hs64", "loud", {"KLLM_ATTN_SPLIT": "2"}, True, "fp32"),
              ("gqa-hs64", "loud", {"KLLM_STAGE_BYTES": "4096", "KLLM_ATTN_SPLIT": "4"}, False, "fp32")]
# int8 weights at their 27 KB stages: T = 256 at hs 64 and T = 192 at hs 128 (Llama-2-7B int8's tile over this cache);
# a split of 2 puts the split edge SP * T inside the sequence
FP8_CASES += [(key, "outliers", {}, calibrated, "int8")
              for key in ("small-int8", "llama2-7b-int8-2l") for calibrated in (False, True)]
FP8_CASES += [("small-int8", "outliers", {"KLLM_ATTN_SPLIT": "2"}, False, "int8"),
              ("llama2-7b-int8-2l", "outliers", {"KLLM_ATTN_SPLIT": "2"}, True, "int8")]
# bf16 weights at their 24 KB stages: T = 192 at hs 128, T = 256 at hs 64
FP8_CASES += [(key, "loud", {}, calibrated, "bf16") for key in ("hs128", "gqa-hs64") for calibrated in (False, True)]
FP8_CASES += [("hs128", "loud", {"KLLM_ATTN_SPLIT": "4"}, True, "bf16")]
assert all(GEOMETRIES[c[0]].head_size % 64 == 0 for c in FP8_CASES)


def report(*parts):
    print("[kv-fp8]", *parts, flush=True)


def fp8_id(c):
    return case_id(c[:3]) + ("-calibrated" if c[3] else "-unit") + ("-bf16w" if c[4] == "bf16" else "")


def make(monkeypatch, shape, w, env=None, kv_cache="fp8", numerics="fast", **kw):
    for name in KNOBS:
        monkeypatch.delenv(name, raising=False)
    for name, value in (env or {}).items():
        monkeypatch.setenv(name, value)
    return Decoder(shape, w, numerics=numerics, kv_cache=kv_cache, **kw)


def fp8_geometry(shape, env, weight_format="fp32"):
    """(T, SP, T_v, stage) of the flash form with an fp8 cache (decode_model_util.engine_geometry): the weight
    format's stage, T = min(stage / hs, 256) & ~31 and T_v the same, the split as fp32's."""
    return engine_geometry(shape, "fast", env, sms(), "fp8", weight_format)


def case_weights(shape, weights, weight_format):
    """(the decoder's weights, the model's): bf16 weights and their exact fp32 widening, else the same dict."""
    w = WEIGHTS[weights](shape, "cuda", 77)
    if weight_format != "bf16":
        return w, w
    w16 = bf16_weights(w)
    return w16, widen_weights(w16)


def ends_for(T, SP, seq_len):
    e = {0, 1, 7, 8, 9, T - 1, T, T + 1, SP * T - 1, SP * T, SP * T + 1, seq_len - 1}
    return sorted(p for p in e if 0 <= p < seq_len)


@pytest.mark.parametrize("key,weights,env,calibrated,weight_format", FP8_CASES, ids=[fp8_id(c) for c in FP8_CASES])
def test_fp8_decode_against_the_model(kllm_lib, monkeypatch, key, weights, env, calibrated, weight_format):
    shape = GEOMETRIES[key]
    w_dec, w = case_weights(shape, weights, weight_format)
    kv_tau, logit_tau = taus(key)
    what = fp8_id((key, weights, env, calibrated, weight_format))
    T, SP = fp8_geometry(shape, env, weight_format)[:2]
    ends = ends_for(T, SP, shape.seq_len)
    toks = sequence(shape.vocab_size, shape.seq_len, 5)
    sin, cos = device_sincos(kllm_lib, shape)
    fixed = shape.group_size == 64
    plain = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends, fixed_point=fixed)
    L, kvh, hs = shape.layer_num, shape.kv_head_num, shape.head_size
    scales = (fp8_kv_scales(plain["k"].float().cpu().numpy(), plain["v"].float().cpu().numpy(), kvh) if calibrated
              else np.ones((2, L, kvh), np.float32))
    model = prefill_ref_fp8(w, shape, toks, 0, sin, cos, scales=scales, tf32=False, logits_at=ends, fixed_point=fixed,
                            rule="decode")
    dec = make(monkeypatch, shape, w_dec, env, kv_scales=scales if calibrated else None,
               weight_format="bf16" if weight_format == "bf16" else "fp32")
    assert dec.engine == "persistent"
    assert dec.attention_geometry == fp8_geometry(shape, env, weight_format), (what, dec.attention_geometry)
    start, logits = 0, {}
    for end in ends:
        dec.generate(0, start, end + 1 - start, teacher=toks[start:end + 1])
        logits[end] = torch.from_numpy(dec.logits()).cuda().double()
        start = end + 1
    k, v = (torch.from_numpy(a).cuda() for a in dec.kv_cache())
    fed = prefill_ref_fp8(w, shape, toks, 0, sin, cos, scales=scales, tf32=False, logits_at=ends, fixed_point=fixed,
                          rule="decode", kv_rows=(k, v))
    # (1) the cache: within one ulp + KV_TAU * rms of the model's rounded rows, and the model's code where that is
    # determined
    worst_kv, decided, total = 0.0, 0, 0
    for which, (name, got, ref) in enumerate((("K", k, fed["k"]), ("V", v, fed["v"]))):
        s = per_head(scales, which, L, kvh, hs, got.device)
        inv = (1.0 / s.float()).double()  # fp32 inverses
        want = fp8_round_rows(ref.float().cpu(), scales, which).to(got.device).double()
        y = (ref.float().double() * inv).float()  # the model's scaled values fp32(x * inv) ...
        code_v = e4m3_rne(y)  # ... and their e4m3 values: want is fp32(code_v * s)
        rms = ref.double().pow(2).mean(-1, keepdim=True).sqrt()
        bound = ulp_e4m3(torch.maximum(code_v.double().abs(), got.double().abs() / s)) * s + kv_tau * rms
        r = float(((got.double() - want).abs() / bound).max())
        worst_kv = max(worst_kv, r)
        assert r <= 1.0, (what, name, r)
        tol = kv_tau * rms * inv
        lo, hi = e4m3_rne((y.double() - tol).float()), e4m3_rne((y.double() + tol).float())
        sure = (lo == hi) & (lo == code_v)
        decided += int(sure.sum())
        total += sure.numel()
        assert torch.equal(got.double()[sure], want[sure]), (what, name)
    # (2) the logits against the model fed the GPU's own cache rows, (3) against the fp32-cache model
    worst_own, worst_plain, rule_dist = 0.0, 0.0, 0.0
    for end in ends:
        own = fed["logits_at"][end]
        rms = float(own.pow(2).mean().sqrt())
        worst_own = max(worst_own, float((logits[end] - own).abs().max()) / (logit_tau * rms))
        rule_dist = max(rule_dist, float((model["logits_at"][end] - plain["logits_at"][end]).abs().max()) / rms)
        worst_plain = max(worst_plain, float((logits[end] - plain["logits_at"][end]).abs().max()) / rms)
    plain_bound = FP8_GAIN * rule_dist + logit_tau
    report(f"{what} T={T} SP={SP}: K/V err / (ulp + tau rms) {worst_kv:.3g}; codes decided and equal "
           f"{decided / total:.4f}; logits err / fast bound vs model on GPU rows {worst_own:.3g}; vs fp32-cache model "
           f"err / rms {worst_plain:.3g} (bound {plain_bound:.3g}, fp8 model's own distance {rule_dist:.3g})")
    assert worst_own <= 1.0, (what, worst_own)
    assert worst_plain <= plain_bound, (what, worst_plain, plain_bound)
    dec.close()


# ---- entries ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small():
    shape = replace(SHAPES["small-int8"], seq_len=640)  # head_size 64
    return shape, synth_weights(shape, "cuda", 2024)


def same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def test_entries_match_stepping(kllm_lib, monkeypatch, small):
    shape, w = small
    toks = sequence(shape.vocab_size, 300, 9)
    sc = np.full((2, shape.layer_num, shape.kv_head_num), 0.01, np.float32)
    a, b = make(monkeypatch, shape, w, kv_scales=sc), make(monkeypatch, shape, w, kv_scales=sc)
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
    d = make(monkeypatch, shape, w, kv_scales=sc)
    d.prompt(toks)
    assert d.generate_until(nxt, len(toks), 40) == ids_step and same(d.logits(), b.logits())
    kd, vd = d.kv_cache()
    ka, va = a.kv_cache()
    assert same(ka, kd) and same(va, vd)
    # every element read back is a code's value times its scale 0.01
    codes = torch.from_numpy(ka[:, :len(toks) + 40]).double() / float(np.float32(0.01))
    assert torch.allclose(codes, e4m3_rne(codes.float()).double(), rtol=1e-6, atol=0)
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
        adj = ref_sampling.penalties(logits, rep_ids=np.array(hist), penalty=penalty,
                                     count_ids=np.array(hist), frequency=freq, presence=pres)
        if ref_sampling.margin(adj, temperature, top_k, seed, p, top_p) > 1e-5:
            assert tok == ref_sampling.sample(adj, temperature, top_k, seed, p, top_p), p
            checked += 1
    report(f"sampled ids checked against the rule: {checked} of 48")
    assert checked >= 40
    dec.close()


@pytest.mark.parametrize("key", ["small-int8", "prefill-hs64"])
def test_batched_prefill_writes_fp8_rows_and_decode_continues(kllm_lib, monkeypatch, key):
    shape = (replace(SHAPES[key], seq_len=640) if key in SHAPES
             else ModelShape("prefill-hs64", 256, 768, 2, 4, 2, 1024, 640))  # fp32, head_size 64
    w = synth_weights(shape, "cuda", 31)
    toks = sequence(shape.vocab_size, 400, 6)
    sin, cos = device_sincos(kllm_lib, shape)
    L, kvh, hs, n = shape.layer_num, shape.kv_head_num, shape.head_size, len(toks)
    plain = prefill_ref(w, shape, toks, 0, sin, cos, tf32=True)
    scales = fp8_kv_scales(plain["k"].float().cpu().numpy(), plain["v"].float().cpu().numpy(), kvh)
    dec = make(monkeypatch, shape, w, kv_scales=scales)
    nxt = dec.prefill_w8(toks) if shape.group_size else dec.prefill_tf32(toks)
    k, v = (torch.from_numpy(a).cuda() for a in dec.kv_cache())
    # the model attends over the GPU's rows (kv_rows): a TF32 difference that moves an element across an e4m3 rounding
    # boundary changes it by one ulp, a step far larger than the prefill bound, which the next layer would carry
    model = prefill_ref_fp8(w, shape, toks, 0, sin, cos, scales=scales, tf32=True, rule="prefill",
                            kv_rows=(k[:, :n], v[:, :n]))
    tau = 5e-2 if shape.group_size else 1e-2  # the prefill bounds (include/kllm_b200.h, tests/test_prefill_*.py)
    worst = 0.0
    for which, (name, got, ref) in enumerate((("K", k[:, :n], model["k"]), ("V", v[:, :n], model["v"]))):
        s = per_head(scales, which, L, kvh, hs, got.device)
        want = fp8_round_rows(ref.float().cpu(), scales, which).to(got.device).double()
        assert torch.allclose(got.double() / s, e4m3_rne((got.double() / s).float()).double(), rtol=1e-6, atol=0), name
        bound = ulp_e4m3(torch.maximum(want.abs(), got.double().abs()) / s) * s + tau * (ref.double().pow(2).mean(-1, keepdim=True).sqrt()
                                                                  + 1e-3)
        worst = max(worst, float(((got.double() - want).abs() / bound).max()))
    report(f"{key} prefill rows err / (ulp + prefill bound) {worst:.3g}")
    assert worst <= 1.0
    lg = torch.from_numpy(dec.logits()).cuda().double()
    report(f"{key} prefill logits err / max|logit| {float((lg - model['logits']).abs().max()) / float(model['logits'].abs().max()):.3g}")
    assert float((lg - model["logits"]).abs().max()) <= 2e-2 * float(model["logits"].abs().max())
    # decode continues over the prefilled fp8 rows, teacher-forced across the next tile edge: each segment end's logits
    # within the fast-mode bound of the model attending over the GPU's prefilled rows (kv_in) and decoded rows (kv_rows)
    assert dec.attention_geometry == fp8_geometry(shape, {}), dec.attention_geometry
    ends = continue_ends(dec.attention_geometry[0], n, shape.seq_len)
    more = sequence(shape.vocab_size, ends[-1] + 1 - n, 16)
    start, logits = n, {}
    for end in ends:
        dec.generate(0, start, end + 1 - start, teacher=more[start - n:end + 1 - n])
        logits[end] = torch.from_numpy(dec.logits()).cuda().double()
        start = end + 1
    k, v = (torch.from_numpy(a).cuda() for a in dec.kv_cache())
    fed = prefill_ref_fp8(w, shape, more, n, sin, cos, scales=scales, tf32=False, logits_at=[e - n for e in ends],
                          fixed_point=shape.group_size == 64, rule="decode", kv_in=(k, v), kv_rows=(k[:, n:], v[:, n:]))
    worst = max(float((logits[e] - fed["logits_at"][e - n]).abs().max())
                / (LOGIT_TAU * float(fed["logits_at"][e - n].pow(2).mean().sqrt())) for e in ends)
    report(f"{key} decode after the prefill, segments {ends}: logits err / fast bound {worst:.3g}")
    assert worst <= 1.0
    dec.close()


def test_bf16_weights_over_the_fp8_cache_equal_fp32_weights_over_the_widened_ones(kllm_lib, monkeypatch):
    shape = replace(SHAPES["small"], name="w16-hs64", dim=256, head_num=4, kv_head_num=2, seq_len=600)
    w16 = bf16_weights(synth_weights(shape, "cuda", 41))
    wide = widen_weights(w16)
    toks = sequence(shape.vocab_size, 300, 2)
    env = {"KLLM_STAGE_BYTES": "24576"}  # one ring geometry for both weight formats
    sc = np.full((2, shape.layer_num, shape.kv_head_num), 0.02, np.float32)
    a = make(monkeypatch, shape, w16, env, weight_format="bf16", kv_scales=sc)
    b = make(monkeypatch, shape, wide, env, kv_scales=sc)
    assert a.attention_geometry == b.attention_geometry
    na, nb = a.prompt(toks), b.prompt(toks)
    assert na == nb and same(a.logits(), b.logits())
    assert a.generate(na, len(toks), 50) == b.generate(nb, len(toks), 50) and same(a.logits(), b.logits())
    for x, y in zip(a.kv_cache(), b.kv_cache()):
        assert same(x, y)
    a.close()
    b.close()


def test_long_context_llama2_7b_int8_agrees_with_the_fp32_cache(kllm_lib, monkeypatch):
    """Llama-2-7B int8 at seq_len 4096: both caches filled by the batched prefill to position 4000 (the fp8 cache at
    scales calibrated on the fp32 cache's rows), then 60 decode steps teacher-forced; logits within LONG_BOUND *
    max|logit| of the fp32 cache's, greedy ids equal wherever the fp32 cache's top-2 margin exceeds twice that.  The
    bound is the size of the fp8 rule itself over 32 layers and 4000 rows (an e4m3 code carries 3 mantissa bits, 16
    times bf16's rounding step; the kernels' own error is held to the fp64 model by the cases above)."""
    shape = replace(SHAPES["llama2-7b-int8"], seq_len=4096)
    w = synth_weights(shape, "cuda", 1234)
    toks = sequence(shape.vocab_size, 4060, 12)
    ref = make(monkeypatch, shape, w, kv_cache="fp32")
    ref.prefill_w8(toks[:4000])
    k, v = ref.kv_cache()
    scales = fp8_kv_scales(k, v, shape.kv_head_num)
    del k, v
    decs = [ref, make(monkeypatch, shape, w, kv_scales=scales)]
    decs[1].prefill_w8(toks[:4000])
    worst = 0.0
    for p in range(4000, 4060, 6):
        out = []
        for d in decs:
            d.generate(0, p, 6, teacher=toks[p:p + 6])
            out.append(d.logits())
        a, b = out
        bound = LONG_BOUND * float(np.abs(a).max())
        worst = max(worst, float(np.abs(a - b).max()) / bound)
        top2 = np.sort(a)[-2:]
        if top2[1] - top2[0] > 2 * bound:
            assert int(np.argmax(a)) == int(np.argmax(b)), p
    report(f"Llama-2-7B int8 pos 4000..4059: |fp8 - fp32 cache| / ({LONG_BOUND} max|logit|) {worst:.3g}")
    assert worst <= 1.0
    for d in decs:
        d.close()


def test_cache_memory_is_a_quarter(kllm_lib, monkeypatch):
    shape = replace(SHAPES["llama2-7b-int8"], layer_num=4, seq_len=4096)
    w = synth_weights(shape, "cuda", 5)
    used = {}
    for c in ("fp32", "fp8"):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        d = make(monkeypatch, shape, w, kv_cache=c)
        used[c] = free0 - torch.cuda.mem_get_info()[0]
        d.close()
    kv = 2 * shape.layer_num * shape.seq_len * shape.kv_dim * 4  # K and V, fp32 bytes
    report(f"create's allocation: fp32 cache {used['fp32'] / 2**20:.1f} MiB, fp8 {used['fp8'] / 2**20:.1f} MiB; "
           f"fp32 K+V {kv / 2**20:.1f} MiB")
    assert abs((used["fp32"] - used["fp8"]) - kv * 3 / 4) <= 8 * 2 ** 20


# ---- refusals --------------------------------------------------------------------------------------------------------
def rc_of(fn):
    """The return code of kllm_decoder_create behind a Decoder(...) call, 0 when it succeeded."""
    try:
        fn().close()
    except KllmError as e:
        return int(str(e).split("failed: ")[1].split()[0])
    return 0


@pytest.mark.parametrize("what", ["exact", "mode-env-exact", "engine-graph", "tp2", "hs32", "hs48", "hs16", "hs256"])
def test_refusals(kllm_lib, monkeypatch, what):
    shape, env, kw = GEOMETRIES["gqa-hs64"], {}, {}
    if what == "exact":
        kw["numerics"] = "exact"
    elif what == "mode-env-exact":
        env["KLLM_MODE"] = "exact"
    elif what == "engine-graph":
        env["KLLM_ENGINE"] = "graph"
    elif what == "hs32":  # the bf16 cache takes it, the fp8 one does not
        shape = SHAPES["small"]
    elif what == "hs48":
        shape = SHAPES["small-hs48"]
    elif what == "hs16":
        shape = GEOMETRIES["hs16"]
    elif what == "hs256":  # head_size 256: the persistent engine's tiles stop at 128; only the graph engine runs it
        shape = replace(SHAPES["small"], name="hs256", dim=512, head_num=2, kv_head_num=2)
    w = synth_weights(shape, "cuda", 3)
    if what == "tp2":
        cb = ALLREDUCE_FN(lambda ctx, buf, n, s: 0)
        rc = rc_of(lambda: Decoder(shape, w, tp_size=2, tp_rank=0, allreduce=cb, numerics="fast", kv_cache="fp8"))
    else:
        rc = rc_of(lambda: make(monkeypatch, shape, w, env, **kw))
    assert rc == -2, (what, rc)
    # and the fp32 cache is not refused where it runs
    if what in ("exact", "mode-env-exact", "engine-graph", "hs32", "hs48", "hs16"):
        make(monkeypatch, shape, w, env, kv_cache="fp32", numerics=kw.get("numerics", "fast")).close()
    if what == "hs32":
        make(monkeypatch, shape, w, env, kv_cache="bf16").close()


@pytest.mark.parametrize("bad", [0.0, -1.0, float("nan"), float("inf")])
def test_bad_scale_is_invalid(kllm_lib, monkeypatch, small, bad):
    shape, w = small
    sc = np.ones((2, shape.layer_num, shape.kv_head_num), np.float32)
    sc[1, -1, -1] = bad
    assert rc_of(lambda: make(monkeypatch, shape, w, kv_scales=sc)) == -1


@pytest.mark.parametrize("cache", ["fp32", "bf16"])
def test_scales_without_the_fp8_cache_are_invalid(kllm_lib, monkeypatch, small, cache):
    shape, w = small
    sc = np.ones((2, shape.layer_num, shape.kv_head_num), np.float32)
    assert rc_of(lambda: make(monkeypatch, shape, w, kv_cache=cache, kv_scales=sc)) == -1


def test_unknown_kv_cache_value_is_invalid(kllm_lib, monkeypatch, small):
    shape, w = small
    d = make(monkeypatch, shape, w, kv_cache="fp32")
    desc = d.desc
    h = ctypes.c_void_p()
    for value in (3, -1):
        desc.kv_cache = value
        assert kllm_lib.kllm_decoder_create(ctypes.byref(desc), None, ctypes.byref(h)) == -1, value
    desc.kv_cache = 2  # the fp8 cache needs its scales: without them the value stays refused
    assert kllm_lib.kllm_decoder_create(ctypes.byref(desc), None, ctypes.byref(h)) == -1
    d.close()


def test_profile_is_refused(kllm_lib, monkeypatch, small):
    shape, w = small
    dec = make(monkeypatch, shape, w)
    stamps = (ctypes.c_uint64 * 65536)()
    g, p = ctypes.c_int32(0), ctypes.c_int32(0)
    assert kllm_lib.kllm_decoder_profile(dec.handle, 1, 0, 2, 0, stamps, 65536, ctypes.byref(g), ctypes.byref(p)) == -2
    dec.close()


# ---- C++ host: KUIPER_KV_CACHE=fp8 ---------------------------------------------------------------------------------
def test_cpp_fp8_kv_cache_matches_the_cabi(kllm_lib, tmp_path, monkeypatch):
    import os
    import subprocess
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
    r = run_decode("llama2", path, "llama", "int8", steps, prompt, env=dict(env, KUIPER_KV_CACHE="fp8"))
    assert r.returncode == 0, r.stderr
    assert [int(x) for x in r.stdout.split()][len(prompt) - 1:] == want
    cmd = [str(ensure_built("llama2")), str(path), "llama", "int8", str(steps), *map(str, prompt), "--kv-cache", "fp8"]
    r2 = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env)
    assert r2.returncode == 0, r2.stderr
    assert r2.stdout.split() == r.stdout.split()
    # without the fast numerics init() fails rather than run an fp32 cache
    env.pop("KUIPER_NUMERICS")
    r3 = run_decode("llama2", path, "llama", "int8", steps, prompt, env=dict(env, KUIPER_KV_CACHE="fp8"))
    assert r3.returncode != 0 and "fp8" in r3.stderr
