"""The fp8 KV cache's rule in the fp64 model (tests/kv_fp8_model.py over tests/prefill_model.py), no GPU.

1. e4m3_rne is torch.float8_e4m3fn's conversion after the clamp to +-448, bit for bit: random values over the whole
   range, exact ties both ways, subnormals (below 2^-6), +-0, saturation at 448 and past it, and non-unit scales.
2. The rule with unit scales and no rounding is the plain model.
3. Negative controls: rounding the current row too, truncating instead of rounding, and reading the codes without
   their scales each move the logits by more than the fast-mode bound the GPU test holds the kernel to.
4. decoder.fp8_kv_scales on a hand-made cache.
"""
import numpy as np
import pytest
import torch

from decode_model_util import LOGIT_TAU, loud_weights
from kv_fp8_model import FP8_MAX, e4m3_codes, e4m3_rne, fp8_round_rows, prefill_ref_fp8, scaled
from prefill_model import prefill_ref

from kuiperllama_b200 import ModelShape
from kuiperllama_b200.decoder import KV_ELEM_BYTES, fp8_kv_scales

SHAPE = ModelShape("fp8-model", 128, 344, 2, 2, 1, 256, 40)  # head_size 64, two query heads per kv head


def torch_e4m3(y):
    """The conversion torch.float8_e4m3fn makes, after the clamp satfinite applies (torch turns overflow into NaN)."""
    y = torch.as_tensor(y).to(torch.float32)
    return y.clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)


def same_codes(ours, y):
    return torch.equal(e4m3_codes(ours), torch_e4m3(y).view(torch.uint8))


def test_e4m3_rne_is_torch_float8_on_random_values():
    g = torch.Generator().manual_seed(5)
    for lo, hi in ((-12.0, 10.0), (-30.0, -5.0)):  # log2 magnitudes: the normal range and deep below the subnormals
        mag = torch.pow(2.0, torch.rand(1 << 18, generator=g) * (hi - lo) + lo)
        sign = torch.where(torch.rand(1 << 18, generator=g) < 0.5, -1.0, 1.0)
        y = (mag * sign).to(torch.float32)
        assert same_codes(e4m3_rne(y), y)


@pytest.mark.parametrize("y", [
    1.0 + 1 / 16, 1.0 + 3 / 16, -(1.0 + 3 / 16),  # ties between 1, 1.125 and 1.25: to even, both ways
    1.0 + 1 / 16 + 2 ** -20, 1.0 + 1 / 16 - 2 ** -20,  # just around a tie
    2 ** -7, 3 * 2 ** -10, 5 * 2 ** -10, 2 ** -10, 2 ** -10 + 2 ** -30, 2 ** -6 - 2 ** -10,  # subnormals and their ties
    2 ** -6, 2 ** -12, -(2 ** -12),  # the smallest normal; a tie at zero -> +-0
    0.0, -0.0,
    448.0, 449.0, 464.0, 465.0, 1e6, -1e6, 3.4e38, float("inf"), float("-inf"),  # saturation at +-448 and past it
])
def test_e4m3_rne_is_torch_float8_at_the_edges(y):
    y = torch.tensor([y], dtype=torch.float32)
    assert same_codes(e4m3_rne(y), y), float(y)


def test_scaled_encoding_is_torch_float8_and_nan_stays_nan():
    g = torch.Generator().manual_seed(6)
    x = (torch.randn(1 << 16, generator=g) * 3).to(torch.float32)
    for s in (1.0, 0.0123, 0.75, 3.0, 1e-4, 7.5e3):
        inv = np.float32(1.0) / np.float32(s)
        want = (x * torch.tensor(inv)).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
        assert torch.equal(e4m3_codes(e4m3_rne(scaled(x, inv))), want.view(torch.uint8)), s
    assert torch.isnan(e4m3_rne(torch.tensor([float("nan")]))).all()
    y = torch.tensor([1.0 + 1 / 16 + 2 ** -20, 1.9])
    assert not torch.equal(e4m3_rne(y, trunc=True), e4m3_rne(y))


@pytest.fixture(scope="module")
def model_inputs():
    from oracle.binding import Oracle
    w = loud_weights(SHAPE, "cpu", 11)
    toks = [int(t) for t in np.random.default_rng(4).integers(0, SHAPE.vocab_size, SHAPE.seq_len)]
    sin, cos = Oracle().sincos(SHAPE.head_size, SHAPE.seq_len, "llama2")
    plain = prefill_ref(w, SHAPE, toks, 0, sin, cos, tf32=False)
    kvh = SHAPE.kv_head_num
    scales = fp8_kv_scales(plain["k"].cpu().numpy(), plain["v"].cpu().numpy(), kvh)
    return w, toks, sin, cos, scales


def test_the_rule_rounds_each_row_at_its_layer_and_heads_scale(model_inputs):
    """With the prefill form every row is rounded: the rows the model attends over are fp8_round_rows of its own rows."""
    w, toks, sin, cos, scales = model_inputs
    seen = []
    import prefill_model
    plain_attention = prefill_model._attention

    def spy(q, k_all, v_all, sp, kv_mul):
        seen.append((k_all.clone(), v_all.clone()))
        return plain_attention(q, k_all, v_all, sp, kv_mul)

    prefill_model._attention = spy
    try:
        r = prefill_ref_fp8(w, SHAPE, toks, 0, sin, cos, scales=scales, tf32=False, rule="prefill")
    finally:
        prefill_model._attention = plain_attention
    assert len(seen) == SHAPE.layer_num
    k = fp8_round_rows(r["k"].cpu(), scales, 0)
    v = fp8_round_rows(r["v"].cpu(), scales, 1)
    for l, (ka, va) in enumerate(seen):
        assert torch.equal(ka.cpu().float().reshape(k[l].shape), k[l]), l
        assert torch.equal(va.cpu().float().reshape(v[l].shape), v[l]), l


def test_negative_controls_move_the_model_past_the_bound(model_inputs):
    w, toks, sin, cos, scales = model_inputs
    ends = list(range(1, SHAPE.seq_len))
    kw = dict(tf32=False, logits_at=ends, scales=scales)
    rule = prefill_ref_fp8(w, SHAPE, toks, 0, sin, cos, rule="decode", **kw)
    controls = {
        "row pos rounded too": prefill_ref_fp8(w, SHAPE, toks, 0, sin, cos, rule="all", **kw),
        "truncated": prefill_ref_fp8(w, SHAPE, toks, 0, sin, cos, rule="decode", trunc=True, **kw),
        "scales ignored": prefill_ref_fp8(w, SHAPE, toks, 0, sin, cos, rule="decode", ignore_scales=True, **kw),
    }
    for name, other in controls.items():
        worst = max(float((other["logits_at"][e] - rule["logits_at"][e]).abs().max())
                    / (LOGIT_TAU * float(rule["logits_at"][e].pow(2).mean().sqrt())) for e in ends)
        print(f"[kv-fp8-model] {name}: worst logit distance / fast-mode bound {worst:.3g}")
        assert worst > 1.0, (name, worst)


def test_fp8_kv_scales_on_a_hand_made_cache():
    L, S, kvh, hs = 2, 5, 3, 4
    k = np.zeros((L, S, kvh * hs), np.float32)
    v = np.zeros_like(k)
    k[0, 2, 0 * hs + 1] = -896.0  # layer 0, head 0: amax 896 (negative)
    k[0, 4, 1 * hs + 3] = 4.48    # layer 0, head 1
    k[1, 0, 2 * hs + 0] = 1.0     # layer 1, head 2; every other K head stays 0 -> scale 1
    v[1, 3, 1 * hs + 2] = 44.8
    sc = fp8_kv_scales(k, v, kvh)
    assert sc.shape == (2, L, kvh) and sc.dtype == np.float32
    want = np.ones((2, L, kvh), np.float32)
    want[0, 0, 0] = np.float32(896.0) / np.float32(448.0)
    want[0, 0, 1] = np.float32(4.48) / np.float32(448.0)
    want[0, 1, 2] = np.float32(1.0) / np.float32(448.0)
    want[1, 1, 1] = np.float32(44.8) / np.float32(448.0)
    assert np.array_equal(sc, want)
    assert np.array_equal(fp8_kv_scales(k.reshape(L, S, kvh, hs), v.reshape(L, S, kvh, hs)), want)
    with pytest.raises(ValueError):
        fp8_kv_scales(k, v)  # three dimensions need the head count


def test_byte_accounting():
    s = ModelShape("x", 4096, 11008, 32, 32, 32, 32000, 4096)
    assert s.kv_bytes_at(4095) == 2 * 32 * 4096 * 4096 * 4
    assert [s.kv_bytes_at(4095, c) * 4 // KV_ELEM_BYTES[c] for c in ("fp32", "bf16", "fp8")] == [s.kv_bytes_at(4095)] * 3
    assert s.kv_bytes_at(4095, "fp8") * 4 == s.kv_bytes_at(4095)
