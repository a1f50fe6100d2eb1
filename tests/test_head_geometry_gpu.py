"""-m gpu: the decode engines at head sizes outside 16, 32, 48, 64 and 128, and at real checkpoints' head counts,
against the fp64 model of tests/prefill_model.py with the harness and bounds of tests/decode_model_util.py.

The persistent engine takes any head_size % 4 == 0 up to 128 in the exact mode, head_size % 16 == 0 in the fast mode
and head_size % 32 == 0 with a bf16 cache.  What depends on the head size: the K-tile producer (one bulk copy per lane
for hs / 4 chunk columns), the flash phase's hs / 16 chunks per quarter head and its partial last 32-lane group in
P.V, the bf16 phase's chunks of 8 dims, and the exact split's V slices of hs / SP floats, which the batched prefill
writes and read_kv converts back.  Each geometry runs, where the engine takes it:
  - the exact mode at every power-of-two split up to the engine's cap, teacher-forced over every position against
    the plain model, and bit for bit against the graph engine (the split changes no FFMA chain);
  - the fast mode at every split up to the cap, and with 32-timestep flash tiles (KLLM_STAGE_BYTES = 32 * hs * 4)
    where a SwiGLU pair of rows still fits such a stage; against the fixed-point model at int8 group 64, else the
    plain model;
  - the bf16 cache against the bf16 model, with test_kv_bf16_gpu.py's bounds;
  - the batched prefill (TF32) in two calls, the second from position 137, on the exact mode at every split, the
    fast mode and the bf16 cache, held to test_prefill_tf32_model_gpu.py's bounds (test_kv_bf16_gpu.py's for the
    bf16 cache), then 16 teacher-forced decode steps over the prefilled rows within the decode bounds;
  - at head_size % 16 != 0, the fast mode's fallback to the graph engine (bit for bit the exact mode there) and its
    refusal when the persistent engine is forced; the bf16 cache's refusal at head_size % 32 != 0;
  - on hs8, hs80 and hs96, greedy free-running exact decoding bit for bit against the reference's CUDA path
    (tests/golden/reference_cuda.json, oracle/reference_golden.py).
Segment ends come from the geometry the engine reports (Decoder.attention_geometry), which every decoder asserts to
be decode_model_util.engine_geometry's: both sides of the first K tile, of the first CTA's second tile and of the
first two V tiles.

Measured worst values (an NVIDIA H100 80GB HBM3 at a 700 W power limit, 132 SMs) are printed with the
[head-geometry] tag; every case stays within the shared constants.
"""
import numpy as np
import pytest
import torch

from decode_model_util import (KV_TAU, KV_TAU_FIRST, LOGIT_TAU, cached_model, clear_cache, compare_engines,
                               device_sincos, fmt, kv_ratios, logit_ratio, make_decoder, run, same_bits)
from kv_bf16_model import bf16_rne, prefill_ref_bf16
from prefill_model import prefill_ref
from test_kv_bf16_gpu import decode_against_the_bf16_model, ulp_bf16
from test_prefill_tf32_model_gpu import KV_TAU as PREFILL_KV_TAU, LOGIT_TAU as PREFILL_LOGIT_TAU

from kuiperllama_b200 import KllmError, ModelShape

pytestmark = pytest.mark.gpu

TAG = "[head-geometry]"
V = 4096  # a reduced vocabulary: the model's logits at every position cost little
# key -> (shape at two layers, weights)
HEADS = {
    "hs8": (ModelShape("hs8-stories260k", 64, 172, 2, 8, 4, V, 512), "loud"),  # stories260K (llama2.c)
    "hs20": (ModelShape("hs20", 160, 432, 2, 8, 2, V, 544), "loud"),
    "hs40": (ModelShape("hs40", 320, 864, 2, 8, 4, V, 544), "loud"),
    "hs100": (ModelShape("hs100", 400, 1088, 2, 4, 2, V, 544), "loud"),
    "hs124": (ModelShape("hs124", 496, 1344, 2, 4, 1, V, 544), "loud"),
    "hs80": (ModelShape("hs80", 640, 1792, 2, 8, 2, V, 1056), "loud"),
    "hs96": (ModelShape("hs96", 768, 2048, 2, 8, 2, V, 1056), "loud"),
    "hs112": (ModelShape("hs112", 896, 2432, 2, 8, 2, V, 1056), "loud"),
    "smollm2-360m-attn": (ModelShape("smollm2-360m-attn", 960, 2560, 2, 15, 5, V, 1056), "loud"),
    "llama3.2-3b-attn": (ModelShape("llama3.2-3b-attn", 3072, 8192, 2, 24, 8, V, 544, flavour="llama3"), "loud"),
    "qwen2.5-3b-attn": (ModelShape("qwen2.5-3b-attn", 2048, 11008, 2, 16, 2, V, 1056, True, flavour="qwen2"),
                        "loud"),
    # int8: at dim 5120 an fp32 SwiGLU pair of rows (40 KB) fits no ring stage, so the fp32 model runs on the graph
    # engine only
    "llama2-13b-attn": (ModelShape("llama2-13b-attn", 5120, 13824, 2, 40, 40, V, 544, group_size=64), "outliers"),
    "hs80-int8-g32": (ModelShape("hs80-int8-g32", 640, 1792, 2, 8, 2, V, 544, group_size=32), "outliers"),
    "hs96-int8-g64": (ModelShape("hs96-int8-g64", 768, 2048, 2, 8, 2, V, 544, group_size=64), "outliers"),
}
REFERENCE_KEYS = ["hs8", "hs80", "hs96"]
PREFILL_CALLS = [137, 120]  # from position 0, then from 137 to 256
DECODE_AFTER_PREFILL = 16


def report(*parts):
    print(TAG, *parts, flush=True)


@pytest.fixture(scope="module", params=list(HEADS))
def geometry(request, kllm_lib):
    """(key, shape, weights, tokens, plain model, fixed-point model or None), the model's logits at every position;
    module scope groups the tests by geometry, so that one is held at a time."""
    key = request.param
    shape, weights = HEADS[key]
    yield (key,) + cached_model(kllm_lib, ("heads", key), shape, weights, range(shape.seq_len))
    clear_cache()


def segment_ends(geom, seq_len):
    """Both sides of the first K tile, of the first CTA's second K tile (SP * T) and of the first two V tiles."""
    T, SP, T_v, _ = geom
    e = {0, 1, 7, 8, 9, T - 1, T, T + 1, SP * T - 1, SP * T, SP * T + 1, T_v - 1, T_v, T_v + 1, 2 * T_v - 1,
         2 * T_v, seq_len - 1}
    return sorted(p for p in e if 0 <= p < seq_len)


def describe(geom):
    T, SP, T_v, stage = geom
    return f"T={T} SP={SP} T_v={T_v} stage={stage}"


def engine_splits(monkeypatch, shape, w, numerics):
    """Every power-of-two split the engine takes for this shape and mode, read from the engine: a KLLM_ATTN_SPLIT
    above its cap is ignored."""
    out = []
    for sp in (1, 2, 4, 8):
        dec = make_decoder(monkeypatch, shape, w, numerics, {"KLLM_ATTN_SPLIT": str(sp)})
        took = dec.attention_geometry[1] == sp
        dec.close()
        if not took:
            break
        out.append(sp)
    return out


def row_bytes(shape, d):
    return d * 4 if shape.group_size == 0 else d + d // shape.group_size * 4


def t32_env(shape):
    """KLLM_STAGE_BYTES giving 32-timestep flash tiles, or None where a SwiGLU pair of rows (W1 and W3, which
    cannot be chunked) does not fit such a stage."""
    stage = 32 * shape.head_size * 4
    return {"KLLM_STAGE_BYTES": str(stage)} if 2 * row_bytes(shape, shape.dim) <= stage else None


# ---- the exact mode -------------------------------------------------------------------------------------------
def test_exact_every_split_against_the_model_and_the_graph_engine(kllm_lib, monkeypatch, geometry):
    key, shape, w, toks, plain, _ = geometry
    make_decoder(monkeypatch, shape, w, "exact", {}).close()  # the default split (geometry asserted)
    out, union = {}, set()
    for sp in engine_splits(monkeypatch, shape, w, "exact"):
        dec = make_decoder(monkeypatch, shape, w, "exact", {"KLLM_ATTN_SPLIT": str(sp)})
        geom = dec.attention_geometry
        ends = segment_ends(geom, shape.seq_len)
        out[sp] = ends, run(f"{key} persistent exact {describe(geom)}", dec, shape, toks, plain, ends, KV_TAU,
                            LOGIT_TAU, tag=TAG)
        union.update(ends)
        dec.close()
    dec = make_decoder(monkeypatch, shape, w, "exact", {}, engine="graph")
    graph = run(f"{key} graph exact", dec, shape, toks, plain, sorted(union), KV_TAU, LOGIT_TAU, tag=TAG)
    dec.close()
    for sp, (ends, res) in out.items():
        compare_engines(f"{key} persistent exact SP={sp} vs graph", shape, ends, res, graph)


# ---- the fast mode, and its fallback ------------------------------------------------------------------------------
def test_fast_mode_against_the_model(kllm_lib, monkeypatch, geometry):
    key, shape, w, toks, plain, fixed = geometry
    if shape.head_size % 16:
        fast_mode_falls_back_to_the_graph_engine(monkeypatch, key, shape, w)
        return
    ref = fixed if fixed is not None else plain
    envs = [{"KLLM_ATTN_SPLIT": str(sp)} for sp in engine_splits(monkeypatch, shape, w, "fast")]
    if t32_env(shape) is not None:
        envs.append(t32_env(shape))
    seen = set()
    for env in envs:
        dec = make_decoder(monkeypatch, shape, w, "fast", env)
        geom = dec.attention_geometry
        if geom in seen:  # the 32-timestep stage may be the default one
            dec.close()
            continue
        seen.add(geom)
        run(f"{key} persistent fast {describe(geom)}", dec, shape, toks, ref, segment_ends(geom, shape.seq_len),
            KV_TAU, LOGIT_TAU, plain=plain if ref is fixed else None, tag=TAG)
        dec.close()


def fast_mode_falls_back_to_the_graph_engine(monkeypatch, key, shape, w):
    """head_size % 16 != 0: the flash phase's quarter heads of 16-byte chunks do not exist, so a fast-mode request
    runs on the graph engine, whose arithmetic is the exact mode's: the same ids, logits and cache bit for bit."""
    steps = 64
    got = {}
    for numerics in ("fast", "exact"):
        dec = make_decoder(monkeypatch, shape, w, numerics, {}, engine=None if numerics == "fast" else "graph")
        assert dec.engine == "graph", (key, numerics, dec.engine)
        got[numerics] = dec.generate(1, 0, steps), dec.logits(), dec.kv_cache()
        dec.close()
    (ids_f, lg_f, (k_f, v_f)), (ids_e, lg_e, (k_e, v_e)) = got["fast"], got["exact"]
    assert ids_f == ids_e and same_bits(lg_f, lg_e), key
    assert same_bits(k_f, k_e) and same_bits(v_f, v_e), key
    with pytest.raises(KllmError, match=r"kllm_decoder_create failed: -2\b"):
        make_decoder(monkeypatch, shape, w, "fast", {}, engine="persistent")
    report(f"{key} fast: graph engine, bit for bit the exact graph decoder over {steps} steps; "
           f"KLLM_ENGINE=persistent refused")


# ---- the bf16 cache -----------------------------------------------------------------------------------------------
def test_bf16_cache_against_the_bf16_model(kllm_lib, monkeypatch, geometry):
    key, shape, w, _, _, _ = geometry
    if shape.head_size % 32:
        with pytest.raises(KllmError, match=r"kllm_decoder_create failed: -2\b"):
            make_decoder(monkeypatch, shape, w, "fast", {}, engine=None, kv_cache="bf16")
        report(f"{key} bf16 cache: refused (head_size {shape.head_size} % 32 != 0)")
        return
    decode_against_the_bf16_model(kllm_lib, monkeypatch, f"{key} bf16", shape, w, {}, KV_TAU, LOGIT_TAU, tag=TAG)


# ---- the batched prefill ------------------------------------------------------------------------------------------
def prefill_modes(monkeypatch, shape, w):
    """(numerics, env, kv_cache) of every persistent form the prefill writes a cache layout for."""
    modes = [("exact", {"KLLM_ATTN_SPLIT": str(sp)}, "fp32")
             for sp in engine_splits(monkeypatch, shape, w, "exact")]
    if shape.head_size % 16 == 0:
        modes.append(("fast", {}, "fp32"))
    if shape.head_size % 32 == 0:
        modes.append(("fast", {}, "bf16"))
    return modes


def test_prefill_against_the_tf32_model_then_decode(kllm_lib, monkeypatch, geometry):
    key, shape, w, toks, _, _ = geometry
    n = sum(PREFILL_CALLS)
    ends = list(np.cumsum(PREFILL_CALLS) - 1)
    sin, cos = device_sincos(kllm_lib, shape)
    models = {}
    for numerics, env, kv_cache in prefill_modes(monkeypatch, shape, w):
        if kv_cache not in models:
            if kv_cache == "bf16":
                models[kv_cache] = prefill_ref_bf16(w, shape, toks[:n], 0, sin, cos, rule="prefill", tf32=True,
                                                    logits_at=ends)
            else:
                models[kv_cache] = prefill_ref(w, shape, toks[:n], 0, sin, cos, tf32=True, logits_at=ends)
        ref = models[kv_cache]
        dec = make_decoder(monkeypatch, shape, w, numerics, env, kv_cache=kv_cache)
        what = f"{key} prefill {numerics} {kv_cache} {describe(dec.attention_geometry)}"
        start = 0
        for count in PREFILL_CALLS:
            chunk = toks[start:start + count]
            nxt = dec.prefill_w8(chunk, start) if shape.group_size else dec.prefill_tf32(chunk, start)
            start += count
            check_prefill_logits(what, dec, nxt, ref["logits_at"][start - 1], kv_cache, shape)
        k, v = dec.kv_cache()
        check_prefill_rows(what, k[:, :n], v[:, :n], ref, kv_cache, shape)
        decode_after_prefill(what, dec, shape, w, toks, n, (k, v), sin, cos, numerics, kv_cache)
        dec.close()


def check_prefill_logits(what, dec, nxt, lref, kv_cache, shape):
    got = torch.from_numpy(dec.logits()).cuda().double()
    if kv_cache == "bf16":  # test_kv_bf16_gpu.py's prefill bound
        bound = 2e-2 * float(lref.abs().max())
    else:
        bound = PREFILL_LOGIT_TAU * float(lref.pow(2).mean().sqrt())
    ratio = float((got - lref).abs().max()) / bound
    report(what, f"logits err / bound {ratio:.3g}")
    assert ratio <= 1.0, (what, ratio)
    top2 = torch.topk(lref, 2).values
    if float(top2[0] - top2[1]) > 2 * bound:
        assert nxt == int(torch.argmax(lref)), what


def check_prefill_rows(what, k, v, ref, kv_cache, shape):
    worst = {}
    for name, got, exp in (("K", k, ref["k"]), ("V", v, ref["v"])):
        got = torch.from_numpy(got).cuda()
        rms = exp.pow(2).mean(-1, keepdim=True).sqrt()
        if kv_cache == "bf16":  # test_kv_bf16_gpu.py's prefill bound: one ulp plus the prefill's
            assert torch.equal(bf16_rne(got), got), (what, name)
            want = bf16_rne(exp).double()
            bound = ulp_bf16(want) + (5e-2 if shape.group_size else 1e-2) * (rms + 1e-3)
        else:
            want = exp
            bound = PREFILL_KV_TAU * rms
        worst[name] = [float(f"{float(r):.3g}") for r in ((got.double() - want).abs() / bound).amax(dim=(1, 2))]
    report(what, f"K / V err / bound per layer {worst}")
    for name, per_layer in worst.items():
        assert max(per_layer) <= 1.0, (what, name, per_layer)


def decode_after_prefill(what, dec, shape, w, toks, n, kv, sin, cos, numerics, kv_cache):
    """DECODE_AFTER_PREFILL teacher-forced steps from position n in two segments, against the model fed the rows
    the prefill cached (so that its TF32 error does not count against the decode bounds)."""
    m = DECODE_AFTER_PREFILL
    fixed = numerics == "fast" and shape.group_size == 64
    seg = [m // 2 - 1, m - 1]
    kv_in = tuple(torch.from_numpy(a).cuda() for a in kv)
    logits = {}
    start = 0
    for end in seg:
        dec.generate(0, n + start, end + 1 - start, teacher=toks[n + start:n + end + 1])
        logits[end] = dec.logits()
        start = end + 1
    k, v = dec.kv_cache()
    got = (k[:, n:n + m], v[:, n:n + m])
    if kv_cache == "bf16":
        rows = tuple(torch.from_numpy(a).cuda() for a in got)
        ref = prefill_ref_bf16(w, shape, toks[n:n + m], n, sin, cos, rule="decode", kv_rows=rows, kv_in=kv_in,
                               tf32=False, logits_at=seg, fixed_point=fixed)
        worst_kv = 0.0
        for name, g, r in (("K", rows[0], ref["k"]), ("V", rows[1], ref["v"])):
            want = bf16_rne(r).double()
            bound = ulp_bf16(want) + KV_TAU * r.pow(2).mean(-1, keepdim=True).sqrt()
            worst_kv = max(worst_kv, float(((g.double() - want).abs() / bound).max()))
        per_layer = {"K / V vs ulp + KV_TAU rms": [float(f"{worst_kv:.3g}")]}
    else:
        ref = prefill_ref(w, shape, toks[n:n + m], n, sin, cos, kv_in=kv_in, tf32=False, logits_at=seg,
                          fixed_point=fixed)
        per_layer = fmt(kv_ratios(got, ref, KV_TAU, KV_TAU_FIRST))
    worst_logit = max(logit_ratio(logits[e], ref["logits_at"][e], LOGIT_TAU) for e in seg)
    report(what, f"then {m} decode steps: logits err / bound {worst_logit:.3g}; K / V err / bound {per_layer}")
    assert worst_logit <= 1.0, (what, worst_logit)
    for name, vals in per_layer.items():
        assert max(vals) <= 1.0, (what, name, vals)


# ---- the reference's CUDA path ------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", REFERENCE_KEYS)
def test_free_running_exact_decode_identical_to_reference_cuda(kllm_lib, monkeypatch, tmp_path, key):
    """Greedy decoding feeding its own output from token 1 over every position: ids and final logits bit for bit
    the reference's (its mha_kernel.cu takes any head_size % 4 == 0), on both engines and at the largest exact
    split."""
    from oracle.reference_golden import Reference
    from test_decoder_gpu import ref_decode

    from kuiperllama_b200 import synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape, _ = HEADS[key]
    w = synth_weights(shape, "cuda", 300 + shape.head_size)
    path = tmp_path / f"{key}.bin"
    write_checkpoint(str(path), shape, w)
    ref = Reference("llama2")
    steps = shape.seq_len
    theirs, lg = ref_decode(ref, path, False, shape.vocab_size, steps)
    cap = engine_splits(monkeypatch, shape, w, "exact")[-1]
    for engine, env in (("persistent", {}), ("persistent", {"KLLM_ATTN_SPLIT": str(cap)}), ("graph", {})):
        dec = make_decoder(monkeypatch, shape, w, "exact", env, engine=engine)
        mine = dec.generate(1, 0, steps)
        what = f"{key} {engine} {env or ''}"
        ref.ids(f"heads/{key}/{steps}/ids", mine, theirs, what)
        ref.bits(f"heads/{key}/{steps}/logits", dec.logits(), lg, f"{what}: logits after {steps} free-running steps")
        dec.close()
    report(f"{key}: {steps} free-running exact steps bit for bit the reference CUDA path (persistent SP 1 and "
           f"SP {cap}, graph)")
