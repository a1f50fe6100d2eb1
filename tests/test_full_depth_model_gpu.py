"""-m gpu: the full-size decoders against the fp64 model at full depth and full context, and caches past 2^31
elements.

Each case builds a decoder at a full checkpoint shape (synthetic weights), fills its cache with the batched prefill
(prefill_w8 or prefill_tf32) to near the end, then teacher-forces decode segments that end on the attention tiles'
edges past that point (the geometry the decoder reports) and on seq_len - 1.  tests/deep_model.py runs only the
checked rows through the layers, one layer's weights in fp64 at a time, each row attending over the decoder's own
cache rows; so the error does not build up along the positions, and a check at position 16 000 is as tight as one at
position 40.  Checked:
  - the logits at every segment end, against the decode step's model (the fast mode's fixed point on int8 weights, the
    plain fp32 model in the exact mode), within LOGIT_TAU_DEEP * rms (Llama-2-7B: LOGIT_TAU), and the greedy id
    wherever the model's top-2 margin exceeds twice that bound;
  - every layer's K / V rows at those positions, within KV_TAU_DEEP * rms (Llama-2-7B: KV_TAU; layer 0: KV_TAU_FIRST),
    plus one element of the cache (a bf16 ulp, or an e4m3 ulp times the scale) over the reduced caches, as
    tests/test_kv_bf16_gpu.py and tests/test_kv_fp8_gpu.py hold them;
  - the prefill's rows at every 97th position and on both sides of its 256-row blocks' edges, and the logits of its
    last row, against the model of its TF32 arithmetic within the prefill's 22-layer constants
    (tests/test_prefill_tf32_model_gpu.py; Llama-2-7B: PRE_TAU_7B), plus one cache element.

Cases: Llama-2-7B int8 at seq_len 4096 on the persistent engine's fast mode over the fp32 cache and the fp8 cache
(scales calibrated on the fp32 cache's rows), and its exact mode; Llama-2-7B with bf16 weights, exact, and fast over the
fp8 cache; Qwen2.5-0.5B at seq_len 16384 (bias, half-split RoPE at theta 1e6, 24 layers) fast over the fp32 and fp8
caches and on the graph engine; TinyLlama-1.1B at seq_len 2048 fast over the bf16 and fp8 caches.  And two synthetic
shapes whose caches reach past 32-bit indices, with the batched prefill writing its rows at the far end: 132 layers over
an fp8 cache of 2.2e9 elements per K / V tensor (past 2^31; the fast mode), and 66 layers over an fp32 cache of 4.4 GB
per tensor (past 2^32 bytes; the exact mode on both engines).  On both, kllm_decoder_copy_prefix copies every row but
the last into a second decoder, and the two step position seq_len - 1 bit for bit alike (in one Batch.step in the exact
mode, which the batch takes).  Rows below the far end's prefill are the cache's zeros, which the model attends over as
the decoder does.  `hs128-long` holds the exact mode's split P.V phase past the probabilities its shared memory holds
(1024 at hidden_dim 1024): there each CTA of a head keeps its own global row, and a row shared by the head's CTAs (each
runs its softmax in place) broke the 66-layer case at position 32560 by 1.1e3 bounds.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, printed with the [deep-model] tag; worst error / bound:
  decode logits             0.409 (qwen2.5-0.5b, graph engine); the greedy id checked at every segment end
  decode K / V, fp32 cache  0.36 (llama2-7b-int8 fast, layer 26); the reduced caches 1.00 (one ulp where the GPU's
                            fp32 value and the model's lie on either side of a rounding boundary)
  prefill K / V             0.47 (llama2-7b-int8, layer 28); 0.42 (qwen2.5-0.5b); the reduced caches 0.953
  prefill last logits       0.43 (llama2-7b-int8)
Llama-2-7B's dim 4096 at 32 layers goes past the 22-layer constants: its decode rows reach 2.16e-5 of their rms and
its logits 2.27e-5 (1.08 and 1.14 of KV_TAU_DEEP and LOGIT_TAU_DEEP), so it is held to KV_TAU and LOGIT_TAU, the
constants of Llama-2-7B at two layers (margins 2.8x and 3.5x); its prefill rows reach 1.41e-2 of their rms (0.70 of
the prefill's 22-layer 2e-2), so they have PRE_TAU_7B = 3e-2 (margin 2.1x).
The module takes about 490 s on that card: 414 s for the other cases together, 78 s for the graph engine over the fp32
cache past 2^32 bytes.  The 7B prefill and kllm_decoder_read_kv's read-backs, 4.3 GB to 17.7 GB, take most of it.
At most 31.0 GiB of device memory is in use.

Sensitivity, each a scratch build of the kernels with one defect, measured as error / bound:
  - fp8 K scale of layer l - 1 read for every layer l >= 2: llama2-7b-int8 fp8 fails, decode logits 2.08e3 and K / V
    28.7.  The two-layer fp8 cases of test_kv_fp8_gpu.py pass, as does its 0.3 max|logit| long-context test (0.604 of
    its bound).
  - the exact mode's K tile read at a 32-bit byte offset, which wraps inside the buffer: big-fp32 fails, logits 22.9 and
    K / V 16.5 in layer 65.  Every other cache is under 2^32 bytes per tensor, where the truncation changes nothing.
  - the last timestep of each position's final flash tile dropped from position 4000 on: llama2-7b-int8 fp32 fails
    (logits 2.11e3), and so do qwen2.5-0.5b fp32 (210) and fp8 (187).
  - the parent commit's shared P.V row: hs128-long fails at position 3007, logits 1.48e3.
"""
import gc
import time
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import (KNOBS, KV_TAU, KV_TAU_DEEP, KV_TAU_FIRST, LOGIT_TAU, LOGIT_TAU_DEEP, clear_cache,
                               device_sincos, engine_geometry, sequence, sms)
from deep_model import sampled_ref
from kv_bf16_model import bf16_rne
from kv_fp8_model import fp8_round_rows, per_head, ulp_e4m3

from kuiperllama_b200 import SHAPES, Batch, Decoder, ModelShape, synth_weights
from kuiperllama_b200.decoder import bf16_weights, fp8_kv_scales

pytestmark = pytest.mark.gpu

# the batched prefill's 22-layer constants (tests/test_prefill_tf32_model_gpu.py KV_TAU_DEEP, LOGIT_TAU_DEEP), and
# Llama-2-7B's at 32 layers (rows 1.41e-2, logits 1.30e-2)
PRE_TAU = 2e-2
PRE_LOGIT_TAU = 2e-2
PRE_TAU_7B = 3e-2
BLOCK = 256  # the batched prefill's rows per pass (run_prefill)

# key: (shape, weight format, prefill start, decode start).  The decode start leaves a tile edge of every geometry
# before seq_len - 1.
MODELS = {
    "llama2-7b-int8": (replace(SHAPES["llama2-7b-int8"], seq_len=4096), "int8", 0, 4000),
    "llama2-7b-bf16w": (replace(SHAPES["llama2-7b"], seq_len=4096), "bf16", 0, 4000),
    "qwen2.5-0.5b": (replace(SHAPES["qwen2.5-0.5b"], seq_len=16384), "fp32", 0, 16100),
    "tinyllama-1.1b": (SHAPES["tinyllama-1.1b"], "fp32", 0, 1700),
    # head_size 128, int8 weights: 132 * 32768 * 512 = 2.2e9 fp8 elements per tensor
    "big-fp8": (ModelShape("big-cache-fp8", 512, 1024, 132, 4, 4, 512, 32768, group_size=64), "int8", 32260, 32560),
    # 66 * 32768 * 512 * 4 bytes = 4.4e9 per tensor
    "big-fp32": (ModelShape("big-cache-fp32", 512, 1024, 66, 4, 4, 512, 32768, group_size=64), "int8", 32260, 32560),
    # the exact mode's split P.V phase past the 1024 probabilities its shared memory holds at hidden_dim 1024
    "hs128-long": (ModelShape("decode-hs128-long", 512, 1024, 3, 4, 2, 2048, 4096), "fp32", 0, 3000),
}
# The decode step's bounds: the 22-layer constants, except at Llama-2-7B's dim 4096, whose 32 layers go past them
# (worst 2.27e-5 of the logits' rms, 2.16e-5 of a row's) and which is held to the constants of Llama-2-7B at two layers
TAUS = {"llama2-7b-int8": (KV_TAU, LOGIT_TAU), "llama2-7b-bf16w": (KV_TAU, LOGIT_TAU)}
PRE_TAUS = {"llama2-7b-int8": PRE_TAU_7B, "llama2-7b-bf16w": PRE_TAU_7B}
BIG_FP8_SCALE = 0.01  # K / V elements of these weights stay within about 3: below 448 * 0.01
# (model, engine, numerics, cache, environment)
CASES = [("llama2-7b-int8", "persistent", "fast", "fp32", {}),
         ("llama2-7b-int8", "persistent", "fast", "fp8", {}),
         ("llama2-7b-int8", "persistent", "exact", "fp32", {}),
         ("llama2-7b-bf16w", "persistent", "exact", "fp32", {}),
         ("llama2-7b-bf16w", "persistent", "fast", "fp8", {}),
         ("qwen2.5-0.5b", "persistent", "fast", "fp32", {}),
         ("qwen2.5-0.5b", "persistent", "fast", "fp8", {}),
         ("qwen2.5-0.5b", "graph", "exact", "fp32", {}),
         ("tinyllama-1.1b", "persistent", "fast", "bf16", {}),
         ("tinyllama-1.1b", "persistent", "fast", "fp8", {}),
         ("big-fp8", "persistent", "fast", "fp8", {}),
         ("big-fp32", "persistent", "exact", "fp32", {}),
         ("big-fp32", "graph", "exact", "fp32", {}),
         ("hs128-long", "persistent", "exact", "fp32", {})]


def case_id(c):
    return "-".join(c[:4]) + "".join(f"-{k[5:].lower()}{v}" for k, v in c[4].items())


def report(*parts):
    print("[deep-model]", *parts, flush=True)


_HELD = {}  # one model's weights at a time, and the fp8 scales calibrated for it
_STATS = {"peak": 0}


def sample_memory():
    free, total = torch.cuda.mem_get_info()
    _STATS["peak"] = max(_STATS["peak"], total - free)


@pytest.fixture(scope="module", autouse=True)
def _clock():
    t0 = time.time()
    yield
    _HELD.clear()
    clear_cache()
    report(f"module wall time {time.time() - t0:.0f} s; peak device memory in use {_STATS['peak'] / 2 ** 30:.1f} GiB "
           f"on {torch.cuda.get_device_name()}")


def weights(key):
    """The decoder's weights of `key` (the model reads the same tensors: bf16 matrices widen exactly)."""
    if _HELD.get("key") != key:
        _HELD.clear()
        clear_cache()
        gc.collect()
        torch.cuda.empty_cache()
        shape, wf = MODELS[key][:2]
        w = synth_weights(shape, "cuda", 1234)
        if wf == "bf16":
            w = bf16_weights(w)
            gc.collect()
            torch.cuda.empty_cache()
        _HELD.update(key=key, w=w)
        sample_memory()
    return _HELD["w"]


def make(monkeypatch, key, engine, numerics, kv_cache, env, scales=None):
    shape, wf = MODELS[key][:2]
    for name in KNOBS:
        monkeypatch.delenv(name, raising=False)
    monkeypatch.setenv("KLLM_ENGINE", engine)
    for name, value in env.items():
        monkeypatch.setenv(name, value)
    dec = Decoder(shape, weights(key), numerics=numerics, kv_cache=kv_cache, kv_scales=scales,
                  weight_format="bf16" if wf == "bf16" else "fp32")
    assert dec.engine == engine
    return dec


def prefill(dec, key, toks):
    shape, _, start, n0 = MODELS[key]
    feed = dec.prefill_w8 if shape.group_size else dec.prefill_tf32
    return feed(toks[start:n0], start)


def calibrated_scales(monkeypatch, key):
    """fp8_kv_scales over the fp32 cache the fast mode's prefill leaves (the rows it will attend over)."""
    if "scales" not in _HELD:  # not left by an fp32-cache case of this model
        if key.startswith("big"):
            shape = MODELS[key][0]
            _HELD["scales"] = np.full((2, shape.layer_num, shape.kv_head_num), BIG_FP8_SCALE, np.float32)
        else:
            dec = make(monkeypatch, key, "persistent", "fast", "fp32", {})
            prefill(dec, key, sequence(MODELS[key][0].vocab_size, MODELS[key][0].seq_len, 5))
            k, v = dec.kv_cache()
            dec.close()
            _HELD["scales"] = fp8_kv_scales(k, v, MODELS[key][0].kv_head_num)
    return _HELD["scales"]


def tail_ends(T, SP, n0, S):
    """Segment ends of the decode from n0: its first two steps, both sides of the first and the last T-timestep tile
    edge after n0 and of the first edge of a CTA's span of SP tiles (if one lies before S), and S - 1."""
    edges = list(range((n0 // T + 1) * T, S, T))
    assert edges, (T, n0, S)
    chosen = {edges[0], edges[-1]} | set([e for e in edges if e % (SP * T) == 0][:1])
    ends = {n0, n0 + 1, S - 1}
    for e in chosen:
        ends |= {e - 1, e, e + 1}
    return sorted(p for p in ends if n0 <= p < S)


def prefill_positions(start, n0):
    """Every 97th row of the prefill, its last, and both sides of each of its 256-row blocks' edges."""
    ps = set(range(start, n0, 97)) | {n0 - 1}
    for c in range(start + BLOCK, n0, BLOCK):
        ps |= {c - 1, c, c + 1}
    return sorted(p for p in ps if start <= p < n0)


def cache_ulp(want, got, kv_cache, scales, which, shape):
    """One element of the cache at the larger magnitude of the two: 0 (fp32), a bf16 ulp, or an e4m3 ulp times the
    scale."""
    if kv_cache == "fp32":
        return torch.zeros_like(want)
    if kv_cache == "bf16":
        m = torch.maximum(want.abs(), got.abs()).clamp_min(2.0 ** -126)
        return torch.pow(2.0, torch.floor(torch.log2(m)) - 7)
    s = per_head(scales, which, shape.layer_num, shape.kv_head_num, shape.head_size, want.device)
    return ulp_e4m3(torch.maximum(want.abs(), got.abs()) / s) * s


def kv_ratios(k, v, model, positions, kv_cache, scales, shape, tau_first, tau):
    """Per-layer worst |got - rounded(model)| / (one cache element + tau * rms(row)) over `positions`, K then V."""
    out = {}
    for which, (name, got_all) in enumerate((("K", k), ("V", v))):
        got = torch.from_numpy(np.ascontiguousarray(got_all[:, positions])).cuda().double()
        ref = model[name.lower()]
        if kv_cache == "fp32":
            want = ref.float().double()
        elif kv_cache == "bf16":
            want = bf16_rne(ref).double()
        else:
            want = fp8_round_rows(ref.float(), scales, which).to(ref.device).double()
        rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
        t = torch.full((ref.shape[0], 1, 1), tau, dtype=torch.float64, device=ref.device)
        t[0] = tau_first
        bound = cache_ulp(want, got, kv_cache, scales, which, shape) + t * rms
        out[name] = [float(x) for x in ((got - want).abs() / bound).amax(dim=(1, 2))]
        del got, want
    return out


def fmt(per_layer):
    return {k: f"max {max(v):.3g} (layer {int(np.argmax(v))}), layer 0 {v[0]:.3g}" for k, v in per_layer.items()}


@pytest.mark.parametrize("key,engine,numerics,kv_cache,env", CASES, ids=[case_id(c) for c in CASES])
def test_full_depth_against_the_model(kllm_lib, monkeypatch, key, engine, numerics, kv_cache, env):
    shape, _, start, n0 = MODELS[key]
    S = shape.seq_len
    w = weights(key)
    scales = calibrated_scales(monkeypatch, key) if kv_cache == "fp8" else None
    what = case_id((key, engine, numerics, kv_cache, env))
    dec = make(monkeypatch, key, engine, numerics, kv_cache, env, scales)
    if engine == "persistent":
        want = engine_geometry(shape, numerics, env, sms(), kv_cache, "bf16" if MODELS[key][1] == "bf16" else "fp32")
        assert dec.attention_geometry == want, (what, dec.attention_geometry, want)
        T, SP = dec.attention_geometry[:2]
    else:
        T, SP = 32, 1  # the graph engine has no tiles: the same ends as a 32-timestep one
    toks = sequence(shape.vocab_size, S, 5)
    t0 = time.time()
    prefill(dec, key, toks)
    pre_logits = torch.from_numpy(dec.logits()).cuda().double()
    fork = key.startswith("big")  # the last position also on a prefix copy
    ends = sorted(set(tail_ends(T, SP, n0, S)) | ({S - 2} if fork else set()))
    ids, logits, s0 = {}, {}, n0
    for end in ends:
        if fork and end == S - 1:
            assert s0 == S - 1
            other = make(monkeypatch, key, engine, numerics, kv_cache, env, scales)
            other.copy_prefix(dec, S - 1)
            if numerics == "exact":  # both in one batch pass (the batch takes the exact mode only)
                batch = Batch([dec, other])
                got = batch.step([toks[S - 1]] * 2, [S - 1] * 2)
                batch.close()
            else:
                got = [d.generate(0, S - 1, 1, teacher=toks[S - 1:])[0] for d in (dec, other)]
            a, b = dec.logits(), other.logits()
            assert got[0] == got[1] and np.array_equal(a.view(np.uint32), b.view(np.uint32)), what
            other.close()
            ids[end] = got[0]
        else:
            ids[end] = dec.generate(0, s0, end + 1 - s0, teacher=toks[s0:end + 1])[-1]
        logits[end] = torch.from_numpy(dec.logits()).cuda().double()
        s0 = end + 1
    sample_memory()
    k, v = dec.kv_cache()
    dec.close()
    if kv_cache == "fp32" and not key.startswith("big") and "scales" not in _HELD:
        _HELD["scales"] = fp8_kv_scales(k, v, shape.kv_head_num)
    t_dec = time.time() - t0
    sin, cos = device_sincos(kllm_lib, shape)

    def rows(l):
        return torch.from_numpy(k[l]), torch.from_numpy(v[l])

    fast = numerics == "fast"
    t0 = time.time()
    dm = sampled_ref(w, shape, ends, [toks[p] for p in ends], sin, cos, rows, "decode",
                     fixed_point=fast and shape.group_size == 64)
    pp = prefill_positions(start, n0)
    pm = sampled_ref(w, shape, pp, [toks[p] for p in pp], sin, cos, rows, "prefill", tf32=True)
    sample_memory()
    t_model = time.time() - t0
    # the decode step
    kv_tau, logit_tau = TAUS.get(key, (KV_TAU_DEEP, LOGIT_TAU_DEEP))
    dkv = kv_ratios(k, v, dm, ends, kv_cache, scales, shape, KV_TAU_FIRST, kv_tau)
    worst_logit, worst_end, greedy = 0.0, None, 0
    for end in ends:
        ref = dm["logits"][end]
        bound = logit_tau * float(ref.pow(2).mean().sqrt())
        r = float((logits[end] - ref).abs().max()) / bound
        if r > worst_logit:
            worst_logit, worst_end = r, end
        top2 = torch.topk(ref, 2).values
        if float(top2[0] - top2[1]) > 2 * bound:
            assert ids[end] == dm["next"][end], (what, end)
            greedy += 1
    # the prefill's rows and its last logits
    pre_tau = PRE_TAUS.get(key, PRE_TAU)
    pkv = kv_ratios(k, v, pm, pp, kv_cache, scales, shape, pre_tau, pre_tau)
    pre_ref = pm["logits"][n0 - 1]
    pre_logit = float((pre_logits - pre_ref).abs().max()) / (PRE_TAUS.get(key, PRE_LOGIT_TAU)
                                                              * float(pre_ref.pow(2).mean().sqrt()))
    del k, v
    report(f"{what} T={T} SP={SP} segments {ends}: decode logits err / bound {worst_logit:.3g} (at {worst_end}), "
           f"greedy ids checked {greedy} of {len(ends)}; K / V err / bound {fmt(dkv)}")
    report(f"{what} prefill rows {pp[0]}..{pp[-1]} ({len(pp)}): K / V err / bound {fmt(pkv)}; last logits err / bound "
           f"{pre_logit:.3g}; decoder {t_dec:.1f} s, model {t_model:.1f} s")
    assert worst_logit <= 1.0, (what, worst_end, worst_logit)
    for name, per_layer in dkv.items():
        assert max(per_layer) <= 1.0, (what, "decode", name, per_layer)
    for name, per_layer in pkv.items():
        assert max(per_layer) <= 1.0, (what, "prefill", name, per_layer)
    assert pre_logit <= 1.0, (what, pre_logit)
