"""-m gpu: the graph engine (csrc/decoder.cu enqueue_step, the decode chain of csrc/verify.cu at one position: gemv.cu,
prefill.cu's RoPE scatter, attention.cu), and both engines at int8 group sizes other than 64, against
tests/prefill_model.py, with the harness and bounds of test_decode_model_gpu.py (tests/decode_model_util.py).

1. Every case of test_decode_model_gpu.py on the graph engine in exact numerics, teacher-forced over every position
   to seq_len - 1: the logits at each segment end and every K / V row of every layer against the model, and both
   bit for bit against the persistent engine's exact mode, which reproduces the same reference order (DESIGN.md
   section 4).
2. Shapes only the graph engine takes, each asserted to land there when no engine is forced: int8 scale rows that
   are not 16-byte multiples (group 32 over dim 288: 36 bytes), groups that span row ends (group 64 over dim 96),
   seq_len % 4 != 0, head_size 160, 188, 192 and 256 (the last two need more than 48 KB of shared memory in the
   attention kernel), and the exporter's golden int8 file (4-byte scale rows).
3. Groups of 32, 96 (the division path), 128 and 256 on shapes both engines take: the persistent engine in exact
   and fast numerics and the graph engine in exact numerics.  The fast mode keeps the exact int8 rows unless the
   group is 64, so its layer-0 rows equal the exact mode's bit for bit and the plain model is its reference.  One
   batched int8 prefill at group 128 against the TF32 model.

Constants: the shared ones of tests/decode_model_util.py.  The worst error each case measured, in units of the
row's (or the logits') rms, on an NVIDIA H100 80GB HBM3 at a 700 W power limit:
    graph engine, the persistent cases: bit for bit the persistent exact mode, so the worst values of
        test_decode_model_gpu.py (exact) hold
    graph-only shapes            K / V layer 0   K / V layer 1   logits
        int8-g32-scale36 outliers    1.43e-6         1.01e-6         8.96e-7
        int8-g64-rowspan synth       6.49e-7         6.42e-7         7.80e-7
        seq1001 loud                 8.20e-7         1.60e-5         1.87e-5
        hs160 loud                   7.08e-7         1.13e-5         1.06e-5
        hs188 loud                   8.71e-7         1.91e-5         2.98e-5   (0.37 of LOGIT_TAU: the worst)
        hs192 loud                   1.31e-6         1.63e-5         1.25e-5
        hs256 loud                   6.77e-7         2.01e-5         2.24e-5
        golden int8                  4.38e-7         4.78e-7         4.36e-7
    other group sizes, exact (both engines) / fast
        g32 outliers                 1.03e-6         1.37e-6 / 1.37e-6   9.9e-7 / 9.9e-7
        g96 outliers                 1.17e-6         1.33e-6 / 1.33e-6   7.5e-7 / 7.3e-7
        g128 synth                   8.5e-7          1.35e-6 / 1.13e-6   1.77e-6 / 1.28e-6
        g256 synth                   7.8e-7          1.90e-6 / 1.57e-6   1.69e-6 / 1.49e-6
    every case stays within half of each shared constant, so none needs its own.
    prefill_w8 at group 128 (both engines): K / V 1.50e-3, logits 1.22e-3, against the TF32 constants 5e-3.
"""
from dataclasses import replace

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from decode_model_util import (CASES, GEOMETRIES, KV_TAU, LOGIT_TAU, cached_model, case_id, clear_cache,
                               compare_engines, device_sincos, edge_ends, flash_geometry, make_decoder, report, run,
                               same_bits, sequence, sms, taus)
from prefill_model import prefill_ref

from kuiperllama_b200 import SHAPES, ModelShape

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _free():
    yield
    clear_cache()


# ---- 1. the persistent cases on the graph engine --------------------------------------------------------------------
@pytest.mark.parametrize("key,weights,env", CASES, ids=[case_id(c) for c in CASES])
def test_graph_engine_against_the_model_and_the_persistent_engine(kllm_lib, monkeypatch, key, weights, env):
    shape = GEOMETRIES[key]
    ends = edge_ends(*flash_geometry(shape, {}, sms()), shape.seq_len)
    shape, w, toks, plain, _ = cached_model(kllm_lib, (key, weights, "ends"), shape, weights, ends)
    kv_tau, logit_tau = taus(key)
    out = {}
    for engine in ("graph", "persistent"):
        dec = make_decoder(monkeypatch, shape, w, "exact", {}, engine=engine)
        out[engine] = run(f"{key} {weights} {engine} exact", dec, shape, toks, plain, ends, kv_tau, logit_tau)
        dec.close()
    compare_engines(f"{key} {weights} graph vs persistent", shape, ends, out["graph"], out["persistent"])


# ---- 2. shapes only the graph engine takes --------------------------------------------------------------------------
def golden_int8(device):
    from kuiperllama_b200.checkpoint import read_checkpoint, to_device
    return to_device(read_checkpoint(str(GOLDEN / "tiny_llama2_int8.bin"), True, "llama2")[1], device)


def golden_int8_shape():
    from kuiperllama_b200.checkpoint import read_checkpoint
    return read_checkpoint(str(GOLDEN / "tiny_llama2_int8.bin"), True, "llama2", name="tiny-llama2-int8")[0]


# key -> (shape, weights, why the persistent engine refuses it)
GRAPH_ONLY = {
    # 6 / 2 heads: head_size 48, GQA 3; 288 / 32 = 9 scales per row: 36-byte scale rows; in_dim 288 and 768 end
    # on partial 128-element chunks
    "int8-g32-scale36": (ModelShape("int8-g32-hs48", 288, 768, 2, 6, 2, 1024, 544, group_size=32), "outliers",
                         "scale rows of 36 bytes"),
    # 3 / 1 heads: head_size 32, GQA 3; 96 % 64 != 0: groups run across row ends
    "int8-g64-rowspan": (ModelShape("int8-g64-rowspan", 96, 160, 2, 3, 1, 512, 544, group_size=64), "synth",
                         "groups that span rows"),
    "seq1001": (replace(SHAPES["small"], name="small-seq1001", seq_len=1001), "loud", "seq_len % 4 != 0"),
    "hs160": (ModelShape("hs160", 480, 1280, 2, 3, 1, 1024, 544), "loud", "head_size > 128"),
    "hs188": (ModelShape("hs188", 376, 1024, 2, 2, 1, 1024, 544), "loud", "head_size > 128"),
    "hs192": (ModelShape("hs192", 576, 1536, 2, 3, 1, 1024, 544), "loud", "head_size > 128"),
    "hs256": (ModelShape("hs256", 512, 1376, 2, 2, 1, 1024, 544), "loud", "head_size > 128"),
    "golden-int8": (None, golden_int8, "scale rows of 4 bytes"),
}


def graph_only_ends(seq_len):
    """Both sides of the attention kernel's 32-timestep value tiles and of its 256 threads, and the end."""
    e = {0, 1, 7, 8, 9, 31, 32, 33, 255, 256, 257, seq_len - 1}
    return sorted(p for p in e if p < seq_len)


@pytest.mark.parametrize("key", list(GRAPH_ONLY))
def test_graph_only_shapes_against_the_model(kllm_lib, monkeypatch, key):
    shape, weights, why = GRAPH_ONLY[key]
    if shape is None:
        shape = golden_int8_shape()
    g = shape.group_size
    if g:
        sizes = {"wq": shape.dim * shape.dim, "wk": shape.kv_dim * shape.dim, "wo": shape.dim * shape.dim,
                 "w1": shape.hidden_dim * shape.dim, "w2": shape.dim * shape.hidden_dim,
                 "wcls": shape.vocab_size * shape.dim}
        assert all(n % g == 0 for n in sizes.values()), (key, sizes)  # whole groups in every tensor
        in_dims = (shape.dim, shape.hidden_dim)
        assert any(d % g or (d // g * 4) % 16 for d in in_dims), key  # what the persistent ring cannot stage
    if key == "int8-g64-rowspan":
        assert shape.dim % g != 0 and shape.hidden_dim % g != 0
    ends = graph_only_ends(shape.seq_len)
    shape, w, toks, plain, _ = cached_model(kllm_lib, ("graph-only", key), shape, weights, ends)
    dec = make_decoder(monkeypatch, shape, w, "exact", {}, engine=None)
    assert dec.engine == "graph", (key, why)
    run(f"{key} graph exact ({why})", dec, shape, toks, plain, ends, KV_TAU, LOGIT_TAU)
    dec.close()


# ---- 3. int8 group sizes other than 64, on both engines -------------------------------------------------------------
# every input length d in {dim, hidden, q_rows}: d % g == 0 and 16-byte scale rows ((d / g) * 4 % 16 == 0)
GROUPS = {
    "g32": (ModelShape("int8-g32", 256, 768, 2, 4, 2, 1024, 544, group_size=32), "outliers"),  # head_size 64
    "g96": (ModelShape("int8-g96", 384, 1152, 2, 4, 2, 1024, 544, group_size=96), "outliers"),  # 96: division
    "g128": (ModelShape("int8-g128", 512, 1536, 2, 8, 4, 1024, 544, group_size=128), "synth"),
    "g256": (ModelShape("int8-g256", 1024, 3072, 2, 8, 2, 1024, 544, group_size=256), "synth"),  # head_size 128
}


@pytest.mark.parametrize("key", list(GROUPS))
def test_group_sizes_on_both_engines_against_the_model(kllm_lib, monkeypatch, key):
    shape, weights = GROUPS[key]
    g = shape.group_size
    for d in (shape.dim, shape.hidden_dim, shape.head_num * shape.head_size):
        assert d % g == 0 and (d // g * 4) % 16 == 0, (key, d)
    T, SP = flash_geometry(shape, {}, sms())
    ends = edge_ends(T, SP, shape.seq_len)
    shape, w, toks, plain, fixed = cached_model(kllm_lib, ("groups", key), shape, weights, ends)
    assert fixed is None  # no fixed point at this group size: the plain model is every mode's reference
    out = {}
    for engine, numerics in (("persistent", "exact"), ("persistent", "fast"), ("graph", "exact")):
        dec = make_decoder(monkeypatch, shape, w, numerics, {}, engine=engine)
        out[engine, numerics] = run(f"{key} {weights} {engine} {numerics} T={T} SP={SP}", dec, shape, toks,
                                    plain, ends, KV_TAU, LOGIT_TAU)
        dec.close()
    exact = out["persistent", "exact"]
    compare_engines(f"{key} graph vs persistent", shape, ends, out["graph", "exact"], exact)
    (ke, ve), (kf, vf) = exact[0], out["persistent", "fast"][0]
    # the fast mode keeps the exact int8 rows at this group size: layer 0 (before any attention) is bit for bit the
    # exact mode's, and flash-decoding's reordered sums show from layer 1 on
    assert same_bits(ke[0], kf[0]) and same_bits(ve[0], vf[0]), key
    assert not same_bits(ke[1], kf[1]) or not same_bits(ve[1], vf[1]), key


# the batched prefill's TF32 bounds (test_prefill_tf32_model_gpu.py: 2 to 3 layers); group 128 measured K / V
# 1.50e-3 and logits 1.22e-3 of their rms
PREFILL_KV_TAU = 5e-3
PREFILL_LOGIT_TAU = 5e-3


@pytest.mark.parametrize("engine", ["graph", "persistent"])
def test_prefill_w8_group_128_against_the_tf32_model(kllm_lib, monkeypatch, engine):
    """kllm_decoder_prefill_w8 at group 128 (dequant_w8's scale index at another group size) to position 256 in
    calls of 1, 255 and 1 positions, against the model with TF32 operands."""
    shape = replace(GROUPS["g128"][0], seq_len=288)
    from kuiperllama_b200 import synth_weights
    w = synth_weights(shape, "cuda", 77)
    toks = sequence(shape.vocab_size, 257, 5)
    sin, cos = device_sincos(kllm_lib, shape)
    calls = [1, 255, 1]
    ref = prefill_ref(w, shape, toks, 0, sin, cos, logits_at=list(np.cumsum(calls) - 1))
    dec = make_decoder(monkeypatch, shape, w, "exact", {}, engine=engine)
    start = 0
    worst = 0.0
    for n in calls:
        nxt = dec.prefill_w8(toks[start:start + n], start)
        start += n
        lref = ref["logits_at"][start - 1]
        bound = PREFILL_LOGIT_TAU * float(lref.pow(2).mean().sqrt())
        ratio = float((torch.from_numpy(dec.logits()).cuda().double() - lref).abs().max()) / bound
        worst = max(worst, ratio)
        assert ratio <= 1.0, (engine, start, ratio)
        top2 = torch.topk(lref, 2).values
        if float(top2[0] - top2[1]) > 2 * bound:
            assert nxt == int(torch.argmax(lref)), (engine, start)
    k, v = dec.kv_cache()
    dec.close()
    kv = {}
    for name, got, exp in (("K", k, ref["k"]), ("V", v, ref["v"])):
        got = torch.from_numpy(got[:, :start]).cuda().double()
        rms = exp.pow(2).mean(-1, keepdim=True).sqrt()
        kv[name] = [round(float(r), 4) for r in ((got - exp).abs() / (PREFILL_KV_TAU * rms)).amax(dim=(1, 2))]
    report(f"prefill_w8 g128 {engine}", f"logits err / bound {worst:.3g}; K / V err / bound per layer {kv}")
    for name, per_layer in kv.items():
        assert max(per_layer) <= 1.0, (engine, name, per_layer)
