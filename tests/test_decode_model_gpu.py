"""-m gpu: the persistent engine's decode step, in both numerics modes, against tests/prefill_model.py.

Row p of the model's causal forward is what a decode step at position p computes.  The exact mode is the plain
fp32 model; the fast mode is the same model with the input of every int8 projection replaced by its 24-bit fixed
point (`fixed_point=True`, a mirror of quantize_input_inplace), and flash-decoding attention, which only reorders
the softmax sums.  Each case teacher-forces one seeded sequence over every position 0 .. seq_len - 1 in segments
that end on the flash tiles' edges, compares the logits at every segment end, and then the K / V cache rows of
every layer at every position.  The edges come from decode_model_util.engine_geometry, and every decoder asserts
that the geometry the engine reports (Decoder.attention_geometry) is that one, so the ends cannot drift off the
engine's tiles unnoticed.  Bounds take the form of test_prefill_tf32_model_gpu.py: each K / V element within
KV_TAU * rms(row), the logits within LOGIT_TAU * rms(logits), and the greedy id equal to the model's argmax
wherever the model's top-2 margin exceeds twice the logit bound.  The fast mode is also measured against the plain
model: that distance is what the fixed point costs.

Geometries: head_size 16, 32 (GQA 3), 48, 64 (Qwen bias and half-split pairs) and 128; the Llama-3 flavour at
Llama-3-8B's attention geometry; int8 small shapes and Llama-2-7B at two layers (the quantiser runs several rounds
per phase, the last one partial, and the dp4a rows end on a partial 512-column step); the Qwen2.5 attention
geometry to position 16383 (8 CTAs per head, many tiles each); TinyLlama-1.1B at 22 layers.  On `small` and `hs128`
the fast mode also runs every split count with flash tiles of 32, 64, 128 and 192 timesteps, and of 256 (one
timestep per consumer thread) on `small` and 160 on `hs128`.

Weights: `synth` (synth_weights), `loud` (scores with std ~5, so the online softmax rescales far from 1, and Wo at
std 1/sqrt(dim), so the attention output reaches the next layer undiluted) and `outliers` (int8: two residual
channels at 300x the embedding scale, an all-zero 64-group in the QKV phase's and the W2 phase's input, and a few
-128 weight bytes).

Constants, with the worst error measured over every case in units of the row's (or the logits') rms, on an NVIDIA
H100 80GB HBM3 at a 700 W power limit.  The fast mode's worst stays within 2x of the exact mode's (it is smaller),
so both modes share each constant.  Layer 0's rows come before any attention, so they have a constant of their
own, tight enough that a quantiser with two digit planes misses it by 20x (tests/test_decode_model.py).
    KV_TAU_FIRST    1e-5  layer 0, every case:  exact 2.47e-6, fast 2.43e-6 (llama2-7b-int8-2l outliers)
    KV_TAU          6e-5  later layers:         exact 2.51e-5 (small-hs48 loud), fast 1.39e-5 (small loud, T 192, SP 2)
    LOGIT_TAU       8e-5                        exact 2.57e-5 (small-hs48 loud), fast 2.08e-5 (small loud, T 256, SP 8)
    KV_TAU_DEEP     2e-5  TinyLlama, 22 layers: exact 6.32e-6, fast 5.24e-6
    LOGIT_TAU_DEEP  2e-5                        exact 5.88e-6, fast 4.94e-6
The fixed point's cost, the fast mode against the plain model: K / V within 6.4e-6 of the row rms and logits within
7.0e-6 of their rms (llama2-7b-int8-2l outliers); 1e-6 to 3e-6 on the synth weights.
"""
import numpy as np
import pytest

from decode_model_util import (CASES, GEOMETRIES, KV_TAU, LOGIT_TAU, cached_model, case_id, clear_cache, edge_ends,
                               flash_geometry, make_decoder, run, sms, split_cap, taus)

pytestmark = pytest.mark.gpu

# The constants, with the worst values above beside them, live in tests/decode_model_util.py: the graph engine's
# test holds its cases to the same ones.


# ---- cases (GEOMETRIES and CASES: tests/decode_model_util.py) -------------------------------------------------------
# (geometry, flash tile T); T = 256 = one timestep per consumer thread only on `small`, where two such stages fit
SWEEP_TILES = [("small", T) for T in (32, 64, 128, 192, 256)] + [("hs128", T) for T in (32, 64, 128, 160, 192)]
SWEEP_SPLITS = [1, 2, 4, 8]


def all_ends(key):
    """Every segment end any case of this geometry uses, for the model's logits_at."""
    shape = GEOMETRIES[key]
    ends = set()
    envs = [c[2] for c in CASES if c[0] == key] + [{}]
    envs += [sweep_env(shape, T, sp) for k, T in SWEEP_TILES if k == key for sp in SWEEP_SPLITS]
    for env in envs:
        ends.update(edge_ends(*flash_geometry(shape, env, sms()), shape.seq_len))
    return sorted(ends)


def sweep_env(shape, T, sp):
    return {"KLLM_STAGE_BYTES": str(T * shape.head_size * 4), "KLLM_ATTN_SPLIT": str(sp)}


@pytest.fixture(scope="module", autouse=True)
def _free():
    yield
    clear_cache()


def model(lib, key, weights):
    """(shape, weights, tokens, plain model, fixed-point model or None); one geometry held at a time."""
    return cached_model(lib, (key, weights), GEOMETRIES[key], weights, all_ends(key))


@pytest.mark.parametrize("key,weights,env", CASES, ids=[case_id(c) for c in CASES])
def test_decode_against_the_model(kllm_lib, monkeypatch, key, weights, env):
    shape, w, toks, plain, fixed = model(kllm_lib, key, weights)
    kv_tau, logit_tau = taus(key)
    T, SP = flash_geometry(shape, env, sms())
    ends = edge_ends(T, SP, shape.seq_len)
    what = f"{key} {weights} {env or ''} T={T} SP={SP}"
    caches = {}
    for numerics in ("exact", "fast"):
        dec = make_decoder(monkeypatch, shape, w, numerics, env if numerics == "fast" else {})
        ref = fixed if numerics == "fast" and fixed is not None else plain
        caches[numerics] = run(f"{what} {numerics}", dec, shape, toks, ref, ends, kv_tau, logit_tau,
                               plain=plain if ref is fixed else None)[0]
        dec.close()
    (ke, ve), (kf, vf) = caches["exact"], caches["fast"]
    same = [np.array_equal(a[l].view(np.uint32), b[l].view(np.uint32)) for a, b in ((ke, kf), (ve, vf))
            for l in range(shape.layer_num)]
    if shape.group_size:
        # the quantiser ran: layer 0's rows differ already
        assert not same[0] and not same[shape.layer_num], what
    else:
        # the fp32 rows keep their order in the fast mode: layer 0 is bit for bit the exact mode's, and what
        # differs from layer 1 on comes from flash-decoding alone
        assert same[0] and same[shape.layer_num], what
        assert not same[1] and not same[shape.layer_num + 1], what


# ids end in the engine's 8 consumer warps
@pytest.mark.parametrize("key,T", SWEEP_TILES, ids=[f"{k}-{T}-8" for k, T in SWEEP_TILES])
def test_fast_decode_tiles_and_splits(kllm_lib, monkeypatch, key, T):
    """The fast mode with flash tiles of T timesteps (KLLM_STAGE_BYTES = T * hs * 4) and every split count, on the
    loud weights."""
    shape, w, toks, plain, _ = model(kllm_lib, key, "loud")
    caches = {}
    for sp in SWEEP_SPLITS:
        assert sp <= split_cap(shape, sms()), (key, sp)
        env = sweep_env(shape, T, sp)
        dec = make_decoder(monkeypatch, shape, w, "fast", env)
        assert dec.attention_geometry[:2] == (T, sp), (key, dec.attention_geometry)
        caches[sp] = run(f"{key} loud fast T={T} SP={sp}", dec, shape, toks, plain,
                         edge_ends(T, sp, shape.seq_len), KV_TAU, LOGIT_TAU)[0]
        dec.close()
    # the split took effect: layer 1's rows (after one layer of split attention) differ between SP = 1 and 4
    assert not np.array_equal(caches[1][0][1].view(np.uint32), caches[4][0][1].view(np.uint32)), (key, T)
