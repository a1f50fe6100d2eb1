"""The bf16 KV cache's rounding rule in the fp64 model (tests/kv_bf16_model.py over tests/prefill_model.py), no GPU.

1. bf16_rne is torch.bfloat16's round to nearest even bit for bit: random values over the whole exponent range,
   exact ties both ways, subnormals, +-0, the overflow to inf and inf itself.
2. The rule's two forms are what they say: with the rounding replaced by the identity both equal the plain model,
   and the decode rule computed for all rows at once equals a decode step per position over the rounded rows.
3. Negative controls: rounding the current row too, or truncating instead of rounding, moves the logits by more
   than the fast-mode bound (decode_model_util.LOGIT_TAU) that the GPU test holds the kernel to, so the GPU test
   can tell the rule from its neighbours.
"""
import numpy as np
import pytest
import torch

from decode_model_util import LOGIT_TAU, loud_weights
from kv_bf16_model import bf16_rne, bf16_trunc, prefill_ref_bf16
from prefill_model import prefill_ref

from kuiperllama_b200 import ModelShape

SHAPE = ModelShape("bf16-model", 128, 344, 2, 4, 2, 256, 40)  # head_size 32, two query heads per kv head


def bits(t):
    return torch.as_tensor(t).to(torch.float32).contiguous().view(torch.int32)


def torch_bf16(t):
    return torch.as_tensor(t).to(torch.float32).to(torch.bfloat16).to(torch.float32)


def from_bits(*u):
    return torch.tensor(np.array(u, dtype=np.uint32).view(np.int32)).view(torch.float32)


def test_bf16_rne_is_torch_bfloat16_on_random_values():
    g = torch.Generator().manual_seed(3)
    u = torch.randint(-(2 ** 31), 2 ** 31 - 1, (1 << 20,), generator=g, dtype=torch.int64).to(torch.int32)
    x = u.view(torch.float32)
    x = x[~torch.isnan(x)]
    assert torch.equal(bits(bf16_rne(x)), bits(torch_bf16(x)))


@pytest.mark.parametrize("u", [
    0x3F808000,  # 1 + 2^-8: a tie, kept bit even -> down
    0x3F818000,  # a tie, kept bit odd -> up
    0xBF818000,  # the same, negative
    0x3F80FFFF, 0x3F807FFF, 0x3F808001,  # just around the tie
    0x00000000, 0x80000000,  # +-0
    0x00000001, 0x00008000, 0x00018000, 0x0000FFFF, 0x807FFFFF, 0x007F8000,  # subnormals, ties among them
    0x7F7FFFFF, 0x7F7F8000, 0x7F7F7FFF,  # the largest floats: to inf, a tie to inf, down
    0x7F800000, 0xFF800000,  # +-inf
])
def test_bf16_rne_is_torch_bfloat16_at_the_edges(u):
    x = from_bits(u)
    assert torch.equal(bits(bf16_rne(x)), bits(torch_bf16(x))), hex(u)


def test_bf16_rne_nan_stays_nan_and_truncation_differs():
    assert torch.isnan(bf16_rne(from_bits(0x7FC00001, 0xFF800001))).all()
    x = from_bits(0x3F818000, 0x3F80FFFF)
    assert not torch.equal(bits(bf16_trunc(x)), bits(bf16_rne(x)))


@pytest.fixture(scope="module")
def model_inputs():
    from oracle.binding import Oracle
    w = loud_weights(SHAPE, "cpu", 11)
    toks = [int(t) for t in np.random.default_rng(4).integers(0, SHAPE.vocab_size, SHAPE.seq_len)]
    sin, cos = Oracle().sincos(SHAPE.head_size, SHAPE.seq_len, "llama2")
    return w, toks, sin, cos


def test_the_rule_without_rounding_is_the_plain_model(model_inputs):
    w, toks, sin, cos = model_inputs
    ends = list(range(SHAPE.seq_len))
    plain = prefill_ref(w, SHAPE, toks, 0, sin, cos, tf32=False, logits_at=ends)
    keep = lambda t: torch.as_tensor(t).to(torch.float32)  # noqa: E731
    for rule in ("decode", "prefill", "all"):
        r = prefill_ref_bf16(w, SHAPE, toks, 0, sin, cos, tf32=False, logits_at=ends, rule=rule, kv_round=keep)
        for e in ends:
            assert torch.allclose(r["logits_at"][e], plain["logits_at"][e], rtol=0, atol=1e-9), (rule, e)


def test_the_decode_rule_is_a_step_over_the_rounded_rows(model_inputs):
    """Row p of the one-call decode model = a decode step at p whose cache holds the rounded rows 0 .. p - 1."""
    w, toks, sin, cos = model_inputs
    ends = list(range(SHAPE.seq_len))
    full = prefill_ref_bf16(w, SHAPE, toks, 0, sin, cos, tf32=False, logits_at=ends, rule="decode")
    k_rows, v_rows = bf16_rne(full["k"]).double(), bf16_rne(full["v"]).double()
    for p in (1, 2, 17, SHAPE.seq_len - 1):
        step = prefill_ref_bf16(w, SHAPE, toks[p:p + 1], p, sin, cos, kv_in=(k_rows, v_rows), tf32=False,
                                rule="decode")
        assert torch.allclose(step["logits"], full["logits_at"][p], rtol=0, atol=1e-9), p


def test_negative_controls_move_the_model_past_the_bound(model_inputs):
    w, toks, sin, cos = model_inputs
    ends = list(range(1, SHAPE.seq_len))
    rule = prefill_ref_bf16(w, SHAPE, toks, 0, sin, cos, tf32=False, logits_at=ends, rule="decode")
    own_row = prefill_ref_bf16(w, SHAPE, toks, 0, sin, cos, tf32=False, logits_at=ends, rule="all")
    trunc = prefill_ref_bf16(w, SHAPE, toks, 0, sin, cos, tf32=False, logits_at=ends, rule="decode",
                             kv_round=bf16_trunc)
    for name, other in (("row pos rounded too", own_row), ("truncated", trunc)):
        worst = max(float((other["logits_at"][e] - rule["logits_at"][e]).abs().max())
                    / (LOGIT_TAU * float(rule["logits_at"][e].pow(2).mean().sqrt())) for e in ends)
        print(f"[kv-bf16-model] {name}: worst logit distance / fast-mode bound {worst:.3g}")
        assert worst > 1.0, (name, worst)
