"""tests/deep_model.py's position-sampled model against prefill_model.prefill_ref, no GPU.

Fed the cache rows a full-prefix prefill_ref run computed (rounded to bf16 or to fp8 codes for those caches, as
kv_bf16_model / kv_fp8_model round them), the sampled model's logits and K / V rows at a spread of positions equal the
full run's to fp64 rounding: the decode step's rule (its own row unrounded, the fast mode's fixed point on int8
weights, the plain fp32 model), and the batched prefill's (its own cached row, TF32 operands).  A model that attends
one row too far or too short, rotates at the wrong position or misses the Qwen bias fails by orders of magnitude.
"""
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import GEOMETRIES, WEIGHTS, sequence
from deep_model import sampled_ref
from kv_bf16_model import bf16_rne, prefill_ref_bf16
from kv_fp8_model import fp8_round_rows, prefill_ref_fp8
from prefill_model import prefill_ref

from kuiperllama_b200.decoder import fp8_kv_scales

N = 150  # positions of the full run
POSITIONS = [0, 1, 7, 31, 32, 63, 64, 96, 127, 128, 149]
TOL = 1e-10  # of the rms: fp64 summation order only (an fp32 rounding flip would be ~1e-7)
# (geometry, weights, cache, rule): the decode step over each cache, the prefill's TF32 rows
CASES = [(key, "loud" if key != "small-int8" else "synth", cache, "decode")
         for key in ("small", "small-qwen", "small-int8", "gqa-hs64") for cache in ("fp32", "bf16", "fp8")
         if cache != "fp8" or GEOMETRIES[key].head_size % 64 == 0]
CASES += [(key, "synth", "fp32", "prefill") for key in ("small", "small-qwen", "small-int8", "gqa-hs64")]


def sincos(shape):
    from oracle.binding import Oracle
    return Oracle().sincos(shape.head_size, shape.seq_len, shape.flavour)


def rel(a, b):
    rms = b.pow(2).mean(-1, keepdim=True).sqrt()
    return float(((a - b).abs() / rms).max())


@pytest.mark.parametrize("key,weights,cache,rule", CASES, ids=["-".join(c) for c in CASES])
def test_sampled_model_is_the_full_model(key, weights, cache, rule):
    shape = replace(GEOMETRIES[key], seq_len=N)
    w = WEIGHTS[weights](shape, "cpu", 77)
    toks = sequence(shape.vocab_size, N, 5)
    sin, cos = sincos(shape)
    tf32 = rule == "prefill"
    fixed = shape.group_size == 64 and not tf32
    kw = dict(tf32=tf32, fixed_point=fixed, logits_at=POSITIONS)
    if cache == "fp32":
        full = prefill_ref(w, shape, toks, 0, sin, cos, **kw)
        rows = (full["k"], full["v"])
    elif cache == "bf16":
        full = prefill_ref_bf16(w, shape, toks, 0, sin, cos, rule=rule, **kw)
        rows = (bf16_rne(full["k"]), bf16_rne(full["v"]))
    else:
        plain = prefill_ref(w, shape, toks, 0, sin, cos, **kw)
        scales = fp8_kv_scales(plain["k"].float().numpy(), plain["v"].float().numpy(), shape.kv_head_num)
        full = prefill_ref_fp8(w, shape, toks, 0, sin, cos, scales=scales, rule=rule, **kw)
        rows = (fp8_round_rows(full["k"], scales, 0), fp8_round_rows(full["v"], scales, 1))
    got = sampled_ref(w, shape, POSITIONS, [toks[p] for p in POSITIONS], sin, cos,
                      lambda l: (rows[0][l], rows[1][l]), rule=rule, tf32=tf32, fixed_point=fixed)
    worst = 0.0
    for name in ("k", "v"):
        worst = max(worst, rel(got[name], full[name][:, POSITIONS]))
    for p in POSITIONS:
        worst = max(worst, rel(got["logits"][p], full["logits_at"][p]))
        assert got["next"][p] == int(torch.argmax(full["logits_at"][p])), p
    print(f"[deep-model] {key} {weights} {cache} {rule}: sampled vs full err / rms {worst:.3g}")
    assert worst <= TOL, worst


def test_one_row_too_many_is_seen():
    """The negative control: the decode rule fed the full run's rows but attending over its cached own row as well
    (the prefill rule, an off-by-one in the decode window on an fp8 cache) moves the logits by far more than TOL."""
    shape = replace(GEOMETRIES["gqa-hs64"], seq_len=N)
    w = WEIGHTS["loud"](shape, "cpu", 77)
    toks = sequence(shape.vocab_size, N, 5)
    sin, cos = sincos(shape)
    plain = prefill_ref(w, shape, toks, 0, sin, cos, logits_at=POSITIONS, tf32=False)
    scales = fp8_kv_scales(plain["k"].float().numpy(), plain["v"].float().numpy(), shape.kv_head_num)
    full = prefill_ref_fp8(w, shape, toks, 0, sin, cos, scales=scales, rule="decode", logits_at=POSITIONS, tf32=False)
    rows = (fp8_round_rows(full["k"], scales, 0), fp8_round_rows(full["v"], scales, 1))
    got = sampled_ref(w, shape, POSITIONS, [toks[p] for p in POSITIONS], sin, cos,
                      lambda l: (rows[0][l], rows[1][l]), rule="prefill")
    worst = max(rel(got["logits"][p], full["logits_at"][p]) for p in POSITIONS)
    assert worst > 1e3 * TOL, worst
    assert np.isfinite(worst)
