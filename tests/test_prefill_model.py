"""CPU checks of tests/prefill_model.py, the fp64 model the batched prefill's GPU tests compare against.

1. tf32_rna against known answers of cvt.rna.tf32.f32 (nearest, ties away from zero, carry into the exponent,
   inf / NaN passed through).
2. With TF32 rounding off, prefill_ref is the plain fp32 model: over the golden checkpoints it must give the
   CPU oracle's K / V cache rows and last logits (oracle/kuiper_oracle.c stepping one position at a time)
   within 1e-5.  fp64 against fp32 arithmetic in other orders differs by a few 1e-7 here (|logits| <= 1.4).
   The same over synthetic int8 checkpoints at groups of 32, 96 and 128, and of 64 over rows of 96 and 160
   elements (groups that span row ends).
3. A prompt modelled in chunks (start_pos > 0 with the earlier rows as kv_in) equals one call.
"""
import numpy as np
import pytest
import torch

from conftest import GOLDEN
from prefill_model import dequant_w8, gemm_ref, prefill_ref, tf32_rna

from kuiperllama_b200 import ModelShape, synth_weights


def bits(*u):
    return torch.tensor(np.array(u, dtype=np.uint32).view(np.int32)).view(torch.float32)


def as_bits(t):
    return [int(v) for v in t.reshape(-1).view(torch.int32).numpy().view(np.uint32)]


@pytest.mark.parametrize("x,expect", [
    (0x3F801000, 0x3F802000),  # 1 + 2^-11: an exact tie, away from zero
    (0xBF801000, 0xBF802000),  # -(1 + 2^-11)
    (0x3F803000, 0x3F804000),  # 1 + 3 * 2^-11: tie above an odd TF32 value (ties-to-even would agree)
    (0x3F805000, 0x3F806000),  # 1 + 5 * 2^-11: tie above an even TF32 value (ties-to-even would go down)
    (0x3F801001, 0x3F802000),  # just above a tie
    (0x3F800FFF, 0x3F800000),  # just below a tie
    (0xBF800FFF, 0xBF800000),
    (0x3F801FFF, 0x3F802000),
    (0x3FFFFFFF, 0x40000000),  # 1.9999999 -> 2.0: the carry leaves the mantissa for the exponent
    (0xBFFFFFFF, 0xC0000000),
    (0x7F7FFFFF, 0x7F800000),  # the largest float rounds to inf
    (0x00000000, 0x00000000),
    (0x80000000, 0x80000000),  # -0 keeps its sign
    (0x00000001, 0x00000000),  # smallest subnormal: down to zero
    (0x00001000, 0x00002000),  # subnormal tie, away from zero
    (0x80001000, 0x80002000),
    (0x007FFFFF, 0x00800000),  # largest subnormal carries into the smallest normal
    (0x7F800000, 0x7F800000),  # inf
    (0xFF800000, 0xFF800000),  # -inf
])
def test_tf32_rna_known_answers(x, expect):
    assert as_bits(tf32_rna(bits(x))) == [expect]


def test_tf32_rna_nan_stays_nan():
    out = tf32_rna(bits(0x7FC00000, 0xFFC00001, 0x7F800001))
    assert torch.isnan(out).all()


def test_tf32_rna_is_nearest_on_random_values():
    """Against a plain statement of the rule: the two TF32 neighbours of x (truncate, then one unit up), pick the
    nearer, the one of larger magnitude on a tie."""
    rng = np.random.default_rng(3)
    x = (rng.standard_normal(100000) * np.exp2(rng.integers(-60, 60, 100000))).astype(np.float32)
    u = x.view(np.uint32)
    lo = (u & ~np.uint32(0x1FFF)).view(np.float32).astype(np.float64)
    hi = ((u & ~np.uint32(0x1FFF)) + np.uint32(0x2000)).view(np.float32).astype(np.float64)
    d_lo, d_hi = np.abs(x - lo), np.abs(hi - x)
    expect = np.where(d_hi <= d_lo, hi, lo)
    assert np.array_equal(tf32_rna(torch.from_numpy(x)).double().numpy(), expect)
    # within half a TF32 unit: relative error at most 2^-11
    assert np.all(np.abs(expect - x) <= np.abs(x) * 2.0 ** -11)


def test_gemm_ref_products_are_exact_and_dequant_rounds_after_the_scale():
    """A TF32 product is exact in fp64, and the int8 weight is rounded after fp32(scale * q), not before."""
    x = bits(0x3F801000, 0x3F7FFFFF)  # 1 + 2^-11 (tie) and 1 - 2^-24
    w = bits(0x3FC01000, 0x3F800000)
    out = gemm_ref(x[None, :], w[None, :])
    assert out.item() == (1 + 2.0 ** -10) * (1.5 + 2.0 ** -10) + 1.0
    q = torch.tensor([[3, -1]], dtype=torch.int8)
    s = bits(0x3DAAB000)  # the scale is a tie; fp32(3 * scale) = 0x3E800400, just above 0.25
    # rounding the scale first would give 0x3E802000 (3 * TF32(scale), rounded again) or 0x3E801000
    assert as_bits(dequant_w8(q, s, 2)) == [0x3E800000, 0xBDAAC000]


GOLDENS = [("tiny_llama2_fp32", False, "llama2", None), ("tiny_llama2_fp32_shared", False, "llama2", None),
           ("tiny_llama2_int8", True, "llama2", None), ("tiny_qwen2file_fp32", False, "llama2", "qwen2file")]


def load(name, quant, flavour, oracle_flavour):
    from kuiperllama_b200.checkpoint import read_checkpoint
    shape, w = read_checkpoint(str(GOLDEN / f"{name}.bin"), quant, flavour, qkv_bias=oracle_flavour == "qwen2file")
    toks = [int(t) for t in np.load(GOLDEN / f"{name}.npz")["tokens"]]
    return shape, w, toks


@pytest.mark.parametrize("name,quant,flavour,oracle_flavour", GOLDENS)
def test_prefill_ref_without_tf32_matches_the_cpu_oracle(oracle, name, quant, flavour, oracle_flavour):
    shape, w, toks = load(name, quant, flavour, oracle_flavour)
    om = oracle.open_model(GOLDEN / f"{name}.bin", quant, oracle_flavour or flavour)
    try:
        for t, tok in enumerate(toks):
            nxt, logits = om.step(tok, t)
        k_o, v_o = (a.copy() for a in om.kv_cache())
    finally:
        om.close()
    sin, cos = oracle.sincos(shape.head_size, shape.seq_len, oracle_flavour or flavour)
    r = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False)
    n = len(toks)
    assert np.abs(r["k"].numpy() - k_o[:, :n]).max() < 1e-5
    assert np.abs(r["v"].numpy() - v_o[:, :n]).max() < 1e-5
    assert np.abs(r["logits"].numpy() - logits).max() < 1e-5
    assert r["next"] == nxt


# int8 checkpoints at group sizes other than the goldens' 64, written with write_checkpoint
INT8_GROUPS = [
    ModelShape("int8-g32", 128, 384, 2, 4, 2, 256, 24, group_size=32),
    ModelShape("int8-g96", 192, 384, 2, 4, 2, 256, 24, group_size=96),  # 96: not a power of two
    ModelShape("int8-g128", 256, 512, 2, 4, 2, 256, 24, group_size=128),
    # 96 % 64 and 160 % 64 != 0: groups run across row ends (over the flattened tensor, as export.py writes them)
    ModelShape("int8-g64-rowspan", 96, 160, 2, 3, 1, 512, 24, group_size=64),
]


@pytest.mark.parametrize("shape", INT8_GROUPS, ids=[s.name for s in INT8_GROUPS])
def test_prefill_ref_at_other_group_sizes_matches_the_cpu_oracle(oracle, tmp_path, shape):
    """dequant_w8's scale index against the oracle's (scales[idx / group_size] over each tensor), stepping every
    position of a synthetic checkpoint."""
    from kuiperllama_b200.checkpoint import write_checkpoint
    w = synth_weights(shape, "cpu", 77)
    path = tmp_path / f"{shape.name}.bin"
    write_checkpoint(str(path), shape, w)
    toks = [int(t) for t in np.random.default_rng(5).integers(0, shape.vocab_size, shape.seq_len)]
    om = oracle.open_model(path, True, "llama2")
    try:
        for t, tok in enumerate(toks):
            nxt, logits = om.step(tok, t)
        k_o, v_o = (a.copy() for a in om.kv_cache())
    finally:
        om.close()
    sin, cos = oracle.sincos(shape.head_size, shape.seq_len, "llama2")
    r = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False)
    assert np.abs(r["k"].numpy() - k_o).max() < 1e-5
    assert np.abs(r["v"].numpy() - v_o).max() < 1e-5
    assert np.abs(r["logits"].numpy() - logits).max() < 1e-5
    assert r["next"] == nxt


@pytest.mark.parametrize("name,quant,flavour,oracle_flavour", GOLDENS)
def test_prefill_ref_in_chunks_equals_one_call(oracle, name, quant, flavour, oracle_flavour):
    shape, w, toks = load(name, quant, flavour, oracle_flavour)
    sin, cos = oracle.sincos(shape.head_size, shape.seq_len, oracle_flavour or flavour)
    for tf32 in (False, True):
        one = prefill_ref(w, shape, toks, 0, sin, cos, tf32=tf32)
        k, v = one["k"][:, :1], one["v"][:, :1]
        last = None
        for a, b in ((0, 1), (1, 6), (6, len(toks))):
            last = prefill_ref(w, shape, toks[a:b], a, sin, cos, kv_in=(k, v), tf32=tf32)
            k, v = torch.cat([k[:, :a], last["k"]], 1), torch.cat([v[:, :a], last["v"]], 1)
        assert torch.equal(k, one["k"]) and torch.equal(v, one["v"])
        assert torch.equal(last["logits"], one["logits"]) and last["next"] == one["next"]


def test_tf32_rounding_changes_the_model():
    """The switch is live: TF32 moves the golden model's rows by far more than fp64 round-off."""
    from oracle.binding import Oracle
    shape, w, toks = load("tiny_llama2_fp32", False, "llama2", None)
    sin, cos = Oracle().sincos(shape.head_size, shape.seq_len, "llama2")
    a = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False)
    b = prefill_ref(w, shape, toks, 0, sin, cos, tf32=True)
    d = float((a["k"] - b["k"]).abs().max() / a["k"].abs().max())
    assert 1e-5 < d < 1e-2, d


def test_one_unit_of_fp32_noise_moves_the_model_as_far_as_the_kernels_differ(monkeypatch):
    """Why the whole-prefill bounds of test_prefill_tf32_model_gpu.py sit near 1e-3 of a row's rms and not near
    fp32 round-off: add +-1 unit in the last place wherever the model rounds to fp32 -- what a correct kernel
    with another summation order does -- and the TF32 roundings it flips move the 3-layer small shape's cache
    rows by about 2e-4 of their rms in layer 0 and 1e-3 to 2e-3 by layer 2, the size of the kernels' measured
    difference.  One row alone (no flip yet) moves by a few 1e-7."""
    from dataclasses import replace

    import prefill_model
    from kuiperllama_b200 import SHAPES, synth_weights
    from oracle.binding import Oracle
    shape = replace(SHAPES["small"], seq_len=352)
    w = synth_weights(shape, "cpu", 77)
    sin, cos = Oracle().sincos(shape.head_size, shape.seq_len, "llama2")
    toks = [int(t) for t in np.random.default_rng(5).integers(0, shape.vocab_size, 255)]
    ref = prefill_ref(w, shape, toks, 0, sin, cos)
    g = torch.Generator().manual_seed(1)

    def f32_with_noise(t):
        u = t.to(torch.float32).view(torch.int32)
        return (u + torch.randint(-1, 2, u.shape, generator=g, dtype=torch.int32)).view(torch.float32).double()

    monkeypatch.setattr(prefill_model, "f32", f32_with_noise)
    noisy = prefill_ref(w, shape, toks, 0, sin, cos)
    for name in ("k", "v"):
        rel = (noisy[name] - ref[name]).abs() / ref[name].pow(2).mean(-1, keepdim=True).sqrt()
        per_layer = [float(r) for r in rel.amax(dim=(1, 2))]
        assert 5e-5 < per_layer[0] < 1e-3 and 5e-4 < per_layer[2] < 5e-3, (name, per_layer)
        assert float(rel[:, 0].max()) < 1e-6, name
