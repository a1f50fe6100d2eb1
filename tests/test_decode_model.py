"""CPU checks of the fast decode mode's model (tests/prefill_model.py, fixed_point=True) and of the bounds that
tests/test_decode_model_gpu.py holds the kernels to.

1. The fixed point (quantize_input_inplace in csrc/megakernel.cu, mirrored by fixed_point_parts): known answers,
   the balanced base-256 digit split over every q in [-2^22, 2^22] and the integer range the dp4a sums stay
   in, and the worst rounding error: 2^-22 of the group maximum, not 2^-23, because the kernel multiplies by
   a rounded reciprocal.
2. Negative controls at the GPU test's constants: a quantiser that keeps two digit planes and two broken flash
   attentions move the model by 10x the bound or more, while +-1 unit of fp32 noise at every store (what a correct
   kernel with another summation order does) stays within half of it.
3. Negative controls for tests/test_graph_engine_model_gpu.py: int8 scale groups restarted at each row or taken
   one group too far move layer 0 by 10x KV_TAU_FIRST or more, and attention capped at head_size 128 moves the
   later layers and the logits by 10x KV_TAU and LOGIT_TAU or more.
"""
import math
from dataclasses import replace

import numpy as np
import pytest
import torch

import prefill_model
from prefill_model import FP_ONE, balanced_digits, fixed_point_parts, fixed_point_value, prefill_ref
from decode_model_util import KV_TAU, KV_TAU_FIRST, LOGIT_TAU, loud_weights, outlier_weights

from kuiperllama_b200 import SHAPES, ModelShape, synth_weights


def f32_bits(*u):
    return torch.tensor(np.array(u, dtype=np.uint32).view(np.float32))


def group(*values):
    g = torch.zeros(64, dtype=torch.float32)
    g[:len(values)] = torch.as_tensor(values, dtype=torch.float32)
    return g


# ---- the quantiser -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gmax", [1.0, 3.7, 1e-3, 6.5e4, 0.4887443])
def test_group_maximum_is_full_scale(gmax):
    step, q = fixed_point_parts(group(gmax, -gmax, gmax / 2, 0.0))
    assert q[0, :4].tolist() == [FP_ONE, -FP_ONE, FP_ONE / 2, 0.0]
    assert float(step) == float(np.float32(np.float32(gmax) * np.float32(2.0 ** -22)))


def test_all_zero_group_has_step_and_digits_zero():
    step, q = fixed_point_parts(torch.cat([group(), group(1.0, -2.0)]))
    assert step[0].item() == 0.0 and bool((q[0] == 0).all())
    assert not torch.isnan(q).any()
    assert fixed_point_value(group()).abs().max().item() == 0.0


def test_power_of_two_maximum_gives_an_exact_step():
    x = group(2.0, 1.5, -1.25, 2.0 ** -20, 3 * 2.0 ** -22)
    step, q = fixed_point_parts(x)
    assert float(step) == 2.0 ** -21
    # every fp32 value that is a multiple of 2^-21 and at most 2 in magnitude is represented exactly
    assert torch.equal(fixed_point_value(x)[:4], x[:4].double())
    assert q[0, 4].item() == 2.0  # 1.5 steps: a tie, rounded to even


def test_balanced_digits_of_every_q():
    q = np.arange(-(1 << 22), (1 << 22) + 1, dtype=np.int64)
    a2, a1, a0 = balanced_digits(q)
    assert np.array_equal(65536 * a2 + 256 * a1 + a0, q)
    assert np.abs(a0).max() <= 128 and np.abs(a1).max() <= 128 and np.abs(a2).max() <= 64
    assert a0.min() == -128 and a1.min() == -128 and a2.min() == -64 and a2.max() == 64


def small_int_to_float(d):
    """The kernel's int32 -> fp32 conversion: the bits of 1.5 * 2^23 + d, minus 1.5 * 2^23 (exact for |d| < 2^22)."""
    return (np.asarray(0x4B400000 + np.asarray(d, np.int64), np.int64).astype(np.uint32).view(np.float32)
            - np.float32(12582912.0))


def test_digit_dot_products_stay_in_the_exact_conversion_range():
    """D_k = sum_i w_i a_k,i over a 64-group: |w| <= 128 (the file format allows -128) and |a_k| <= 128, so
    |D_k| <= 64 * 128 * 128 = 2^20, inside the 2^22 that small_int_to_float converts exactly."""
    bound = 64 * 128 * 128
    assert bound == 1 << 20 and bound < 1 << 22
    w = np.full(64, -128, np.int64)
    for digits in (np.full(64, -128, np.int64), np.full(64, 127, np.int64)):
        d = int(w @ digits)
        assert abs(d) <= bound
    d = np.array([-(1 << 20), (1 << 20), -(1 << 22) + 1, (1 << 22) - 1, 0, -1, 12345], np.int64)
    assert np.array_equal(small_int_to_float(d).astype(np.int64), d)
    # the sums the kernel forms from the digits of random q and weights of the whole int8 range
    rng = np.random.default_rng(1)
    q = rng.integers(-(1 << 22), (1 << 22) + 1, (4096, 64))
    w = rng.integers(-128, 128, (4096, 64))
    for a in balanced_digits(q):
        dk = (w * a).sum(1)
        assert np.abs(dk).max() <= bound
        assert np.array_equal(small_int_to_float(dk).astype(np.int64), dk)


# a group whose second element lands 1.64 * 2^-23 of the group maximum from its fixed-point value
OVER_HALF_STEP = (0xBEFA3CB1, 0xBEF2CDCF)


def rounding_error(x):
    """|step * q - x| / gmax per element of x [groups, 64], in fp64."""
    step, q = fixed_point_parts(x)
    xd = x.double().reshape(q.shape)
    gmax = xd.abs().amax(-1, keepdim=True)
    return ((step.double() * q.double() - xd).abs() / gmax.clamp_min(1e-300)).reshape(x.shape)


def test_rounding_error_is_within_2_pow_minus_22_of_the_group_maximum():
    rng = np.random.default_rng(2)
    n = 20000
    x = (rng.standard_normal((n, 64)) * np.exp(rng.uniform(-5, 5, (n, 1)))).astype(np.float32)
    # adversarial: elements half a step from the grid, ties included, and maxima just under a power of two
    gmax = np.exp(rng.uniform(-5, 5, n)).astype(np.float32)
    k = rng.integers(-(1 << 22), 1 << 22, (n, 63))
    adv = np.concatenate([gmax[:, None], ((k + 0.5) * (gmax[:, None].astype(np.float64) / FP_ONE))], 1)
    near_pow2 = np.float32(np.nextafter(np.float32(1.0), np.float32(0.0)))
    adv[:64, 0] = near_pow2 * np.exp2(np.arange(-32, 32))
    x = torch.from_numpy(np.concatenate([x, adv.astype(np.float32)]))
    err = rounding_error(x)
    worst = float(err.max()) * 2 ** 22
    assert worst <= 1.0, worst
    # the bound is not 2^-23: the reciprocal's rounding moves x * inv by more than half a unit
    assert float(err.max()) > 2.0 ** -23
    pinned = rounding_error(torch.cat([f32_bits(*OVER_HALF_STEP), torch.zeros(62)]))
    assert 2.0 ** -23 < float(pinned[1]) <= 2.0 ** -22, float(pinned[1]) * 2 ** 23


# ---- negative controls at the GPU test's constants ------------------------------------------------------------------
def sincos(shape):
    from oracle.binding import Oracle
    return Oracle().sincos(shape.head_size, shape.seq_len, shape.flavour)


def tokens(shape, n, seed=5):
    return [int(t) for t in np.random.default_rng(seed).integers(0, shape.vocab_size, n)]


def kv_rel(a, b):
    """Per-layer worst |a - b| / rms(row of b), for K and V together."""
    worst = []
    for l in range(b["k"].shape[0]):
        r = 0.0
        for name in ("k", "v"):
            rms = b[name][l].pow(2).mean(-1, keepdim=True).sqrt()
            r = max(r, float(((a[name][l] - b[name][l]).abs() / rms).max()))
        worst.append(r)
    return worst


def logit_rel(a, b):
    return max(float((a["logits_at"][i] - b["logits_at"][i]).abs().max() / b["logits_at"][i].pow(2).mean().sqrt())
               for i in b["logits_at"])


def test_two_digit_planes_move_the_first_layer_by_ten_bounds(monkeypatch):
    """(a) A quantiser that loses its lowest digit plane (16-bit fixed point, exact to 2^-15 of the group maximum)
    moves small-int8's layer-0 V rows by >= 10 KV_TAU_FIRST (about 20)."""
    shape = replace(SHAPES["small-int8"], seq_len=96)
    w = synth_weights(shape, "cpu", 77)
    sin, cos = sincos(shape)
    toks = tokens(shape, 96)
    ends = list(range(0, 96, 8))
    ref = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, fixed_point=True, logits_at=ends)

    def two_planes(x):
        step, q = fixed_point_parts(x)
        a2, a1, _ = balanced_digits(q.to(torch.int64))
        return (step.double() * (65536 * a2 + 256 * a1).double()).reshape(x.shape)

    monkeypatch.setattr(prefill_model, "fixed_point_value", two_planes)
    coarse = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, fixed_point=True, logits_at=ends)
    v0 = float(((coarse["v"][0] - ref["v"][0]).abs() / ref["v"][0].pow(2).mean(-1, keepdim=True).sqrt()).max())
    dlogit = max(float((coarse["logits_at"][i] - ref["logits_at"][i]).abs().max()) for i in ends)
    print(f"two digit planes: layer-0 V moves {v0 / KV_TAU_FIRST:.3g} KV_TAU_FIRST; logits move {dlogit:.3g} "
          f"absolute ({dlogit / 1e-4:.3g} of the 1e-4 that test_fast_numerics_within_north_star_tolerance allows)")
    assert v0 >= 10 * KV_TAU_FIRST, v0 / KV_TAU_FIRST


def attention_dropping_tile_ends(T):
    """Causal attention that skips the last timestep of every T-timestep tile of the cache (the current
    position, folded in from registers by the kernel, is kept)."""
    def attention(q, k_all, v_all, start_pos, kv_mul, max_bytes=None):
        n, heads, hs = q.shape
        P = start_pos + n
        k = k_all[:P].repeat_interleave(kv_mul, dim=1)
        v = v_all[:P].repeat_interleave(kv_mul, dim=1)
        s = torch.einsum("nhd,phd->hnp", q, k) / math.sqrt(hs)
        pos = torch.arange(start_pos, P)[:, None]
        t = torch.arange(P)[None, :]
        drop = (t > pos) | ((t < pos) & (t % T == T - 1))
        o = torch.einsum("hnp,phd->nhd", torch.softmax(s.masked_fill(drop[None], float("-inf")), -1), v)
        return prefill_model.f32(o)
    return attention


def attention_merging_without_rescale(split):
    """Flash attention whose partials over `split` interleaved runs of timesteps are merged as num = sum num_s,
    den = sum den_s, each taken relative to its own maximum: the exp(m_s - M) rescale left out."""
    def attention(q, k_all, v_all, start_pos, kv_mul, max_bytes=None):
        n, heads, hs = q.shape
        P = start_pos + n
        k = k_all[:P].repeat_interleave(kv_mul, dim=1)
        v = v_all[:P].repeat_interleave(kv_mul, dim=1)
        s = torch.einsum("nhd,phd->hnp", q, k) / math.sqrt(hs)
        pos = torch.arange(start_pos, P)[:, None]
        t = torch.arange(P)[None, :]
        num, den = 0.0, 0.0
        for part in range(split):
            keep = (t <= pos) & (t % split == part)
            sp = s.masked_fill(~keep[None], float("-inf"))
            m = sp.amax(-1, keepdim=True)
            e = torch.where(keep[None], torch.exp(sp - torch.where(torch.isfinite(m), m, 0.0)), 0.0)
            num = num + torch.einsum("hnp,phd->nhd", e, v)
            den = den + e.sum(-1).permute(1, 0)[..., None]
        return prefill_model.f32(num / den)
    return attention


def loud_small():
    shape = replace(SHAPES["small"], seq_len=160)
    return shape, loud_weights(shape, "cpu", 77), sincos(shape), tokens(shape, 160)


def test_reference_attention_of_the_controls_is_the_model():
    """With nothing dropped (a tile longer than the sequence) and one part, the controls' attention is the
    model's own: what they change is what they break, nothing else."""
    shape, w, (sin, cos), toks = loud_small()
    ref = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False)
    for att in (attention_dropping_tile_ends(10 ** 9), attention_merging_without_rescale(1)):
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(prefill_model, "_attention", att)
            same = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False)
        assert max(kv_rel(same, ref)) < 1e-6


@pytest.mark.parametrize("broken", ["drop-tile-ends", "merge-without-rescale"])
def test_broken_flash_attention_moves_the_model_by_ten_bounds(monkeypatch, broken):
    """(b) On the loud weights, a flash attention that drops the last timestep of every 32-timestep tile, or
    merges two partials without the exp(m_s - M) rescale, moves the cache rows by >= 10 KV_TAU."""
    shape, w, (sin, cos), toks = loud_small()
    ref = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False)
    att = attention_dropping_tile_ends(32) if broken == "drop-tile-ends" else attention_merging_without_rescale(2)
    monkeypatch.setattr(prefill_model, "_attention", att)
    bad = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False)
    per_layer = kv_rel(bad, ref)
    print(f"{broken}: K / V move {[round(r / KV_TAU, 1) for r in per_layer]} KV_TAU per layer")
    assert per_layer[0] == 0.0  # layer 0's rows come before any attention
    assert max(per_layer) >= 10 * KV_TAU


@pytest.mark.parametrize("case", ["small-loud", "small-int8-fixed-point", "small-int8-outliers-fixed-point"])
def test_one_unit_of_fp32_noise_stays_within_half_the_bound(monkeypatch, case):
    """(c) +-1 unit in the last place wherever the model rounds to fp32 -- what a correct kernel with another
    summation order does -- moves the cache rows by at most KV_TAU / 2 and the logits by at most LOGIT_TAU / 2:
    the bounds are not tighter than a correct reordering.  Layer 0 against KV_TAU_FIRST / 2."""
    if case == "small-loud":
        shape, w, (sin, cos), toks = loud_small()
        fixed = False
    else:
        shape = replace(SHAPES["small-int8"], seq_len=96)
        w = (outlier_weights if "outliers" in case else synth_weights)(shape, "cpu", 77)
        (sin, cos), toks, fixed = sincos(shape), tokens(shape, 96), True
    ends = list(range(0, shape.seq_len, 16)) + [shape.seq_len - 1]
    ref = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, fixed_point=fixed, logits_at=ends)
    g = torch.Generator().manual_seed(1)

    def f32_with_noise(t):
        t = t.to(torch.float32)
        u = t.view(torch.int32) + torch.randint(-1, 2, t.shape, generator=g, dtype=torch.int32)
        return torch.where(t == 0, t, u.view(torch.float32)).double()  # a zero stays zero (the all-zero groups)

    monkeypatch.setattr(prefill_model, "f32", f32_with_noise)
    noisy = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, fixed_point=fixed, logits_at=ends)
    per_layer, logits = kv_rel(noisy, ref), logit_rel(noisy, ref)
    print(f"{case}: +-1 ulp moves K / V by {per_layer[0] / KV_TAU_FIRST:.3g} KV_TAU_FIRST in layer 0, "
          f"{[round(r / KV_TAU, 3) for r in per_layer[1:]]} KV_TAU after, logits by {logits / LOGIT_TAU:.3g} LOGIT_TAU")
    assert per_layer[0] <= KV_TAU_FIRST / 2 and max(per_layer[1:]) <= KV_TAU / 2 and logits <= LOGIT_TAU / 2


# ---- negative controls for the graph engine's shapes and other group sizes ------------------------------------------
def dequant_groups_per_row(q, scales, group_size, tf32=True):
    """Groups restarted at each row: element c of row r takes scale r * (K / group) + c / group (integer division),
    what a kernel indexing the scales per row computes, in place of one index over the flattened tensor."""
    q = torch.as_tensor(q)
    n, k = q.shape
    s = torch.as_tensor(scales).to(torch.float32).reshape(-1)
    idx = torch.arange(n)[:, None] * (k // group_size) + torch.arange(k)[None, :] // group_size
    w = s[idx] * q.to(torch.float32)
    return prefill_model.tf32_rna(w) if tf32 else w


def dequant_next_group(q, scales, group_size, tf32=True):
    """The scale index one group too far (the last group keeps its own scale)."""
    q = torch.as_tensor(q)
    n, k = q.shape
    s = torch.as_tensor(scales).to(torch.float32).reshape(-1)
    idx = (torch.arange(n * k) // group_size + 1).clamp(max=s.numel() - 1).reshape(n, k)
    w = s[idx] * q.to(torch.float32)
    return prefill_model.tf32_rna(w) if tf32 else w


MODEL_ATTENTION = prefill_model._attention


def attention_capped_at_128(q, k_all, v_all, start_pos, kv_mul, max_bytes=1 << 28):
    """Attention over the first 128 dimensions of each head only, the output zero beyond them: a kernel whose
    output chains and score loops stop at 128."""
    out = torch.zeros_like(q)
    out[..., :128] = MODEL_ATTENTION(q[..., :128].contiguous(), k_all[..., :128].contiguous(),
                                     v_all[..., :128].contiguous(), start_pos, kv_mul, max_bytes)
    return out


CONTROL_SHAPES = {
    # the graph-only int8 shapes of test_graph_engine_model_gpu.py at 32 positions
    "rowspan": ModelShape("int8-g64-rowspan", 96, 160, 2, 3, 1, 512, 32, group_size=64),
    "g32": ModelShape("int8-g32-hs48", 288, 768, 2, 6, 2, 1024, 32, group_size=32),
    "hs192": ModelShape("hs192", 576, 1536, 2, 3, 1, 1024, 32),
    "hs128": ModelShape("hs128", 256, 688, 2, 2, 1, 512, 32),
}


def control_model(key, seq=32):
    shape = CONTROL_SHAPES[key]
    w = (synth_weights if shape.group_size else loud_weights)(shape, "cpu", 77)
    return shape, w, sincos(shape), tokens(shape, seq), list(range(0, seq, 4)) + [seq - 1]


@pytest.mark.parametrize("key,patch,fn", [("g32", "dequant_w8", dequant_groups_per_row),
                                          ("hs128", "_attention", attention_capped_at_128)])
def test_controls_equal_the_model_where_nothing_differs(key, patch, fn):
    """Groups per row are the flattened groups when the row length is a multiple of the group, and a cap at 128
    does nothing at head_size 128: the controls below break only what they name."""
    shape, w, (sin, cos), toks, ends = control_model(key)
    ref = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(prefill_model, patch, fn)
        same = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends)
    assert max(kv_rel(same, ref)) == 0.0 and logit_rel(same, ref) == 0.0


@pytest.mark.parametrize("broken,key", [("groups-per-row", "rowspan"), ("next-group", "g32"),
                                        ("next-group", "rowspan"), ("head-size-capped", "hs192")])
def test_broken_graph_engine_shapes_move_the_model_by_ten_bounds(monkeypatch, broken, key):
    """Scale groups restarted at each row or taken one group too far move layer 0's K / V rows (before any
    attention) by >= 10 KV_TAU_FIRST; attention capped at head_size 128 moves the later layers' rows by >= 10
    KV_TAU and the logits by >= 10 LOGIT_TAU, leaving layer 0 as it was."""
    shape, w, (sin, cos), toks, ends = control_model(key)
    ref = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends)
    if broken == "head-size-capped":
        monkeypatch.setattr(prefill_model, "_attention", attention_capped_at_128)
    else:
        fn = dequant_groups_per_row if broken == "groups-per-row" else dequant_next_group
        monkeypatch.setattr(prefill_model, "dequant_w8", fn)
    bad = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends)
    per_layer, logits = kv_rel(bad, ref), logit_rel(bad, ref)
    print(f"{broken} on {key}: K / V move {per_layer[0] / KV_TAU_FIRST:.3g} KV_TAU_FIRST in layer 0, "
          f"{[round(r / KV_TAU, 1) for r in per_layer[1:]]} KV_TAU after, logits {logits / LOGIT_TAU:.3g} LOGIT_TAU")
    if broken == "head-size-capped":
        assert per_layer[0] == 0.0
        assert max(per_layer[1:]) >= 10 * KV_TAU and logits >= 10 * LOGIT_TAU
    else:
        assert per_layer[0] >= 10 * KV_TAU_FIRST
