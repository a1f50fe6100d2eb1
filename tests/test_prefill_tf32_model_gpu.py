"""-m gpu: the batched prefill against tests/prefill_model.py, an fp64 model of the same TF32 arithmetic.

test_prefill_gpu.py and test_prefill_int8_gpu.py hold the prefill to the exact stepping path, with bounds wide
enough for TF32 itself (5e-2 of a row's rms).  The model here rounds the GEMM operands to TF32 exactly as the
kernels do (cvt.rna) and rounds to fp32 wherever the kernels store fp32, so what remains is fp32 accumulation
order, and the bounds below are orders of magnitude tighter.  They catch what TF32 noise hides: truncation in
place of rounding, a wrong eps, a RoPE index, a causal window off by one, a misplaced V slice.

GEMM bound.  A TF32 x TF32 product has 22 significant bits, so it is exact in fp32 and in fp64; the only error
of out[t, n] is the rounding of the fp32 sums that add up the K products x~_k w~_k.  With relative rounding
error u per addition and K / 8 additions into the accumulator (one m64nNk8 wgmma per 8 columns of K), the worst
case is (K / 8) * u * S, S = sum_k |x~_k w~_k|.  That assumes every rounding at its maximum and of one sign; the
measured error grows like sqrt(K) instead, as independent roundings do, and NVIDIA does not document the
accumulator's rounding, so the bound is |out - gemm_ref| <= TAU_GEMM * sqrt(K) * S with TAU_GEMM = 2^-23 (one
unit of fp32 truncation).  Measured worst error / bound over every shape below: 0.51 for kllm_gemm_tf32 (K = 4,
T = 513, N = 128) and 0.25 for kllm_gemm_w8_tf32 (K = 64): a margin of 2x.  A kernel that leaves the token tile
unrounded (the tensor core then truncates it) exceeds the bound 59x at K = 4 and 815x at K = 28.

Whole-prefill bound.  Two correct fp32 computations of a row differ in the last bits (fp32 summation order, the
device's rsqrtf / expf, a fused multiply-add).  A one-unit fp32 difference in an activation sometimes flips its
rounding to TF32 in the next GEMM, and that operand then moves by up to 2^-11 of itself; these flips, not the
accumulation order, dominate after the first GEMM, and they ride on the residual stream through the layers.
tests/test_prefill_model.py shows the model moving by the same amount when +-1 unit of noise is added wherever it
rounds to fp32.  So each K / V element is held to KV_TAU * rms(row) and the last logits to
LOGIT_TAU * rms(logits), the 22-layer TinyLlama case to its own constants, and the next id must agree when the
model's top-2 margin exceeds twice the logit bound.  Measured worst ratios are beside the constants.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit.
"""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from gpu_util import ptr, sync
from prefill_model import dequant_w8, gemm_abs_ref, gemm_ref, prefill_ref, tf32_rna

pytestmark = pytest.mark.gpu

KLLM_E_INVALID = -1

TAU_GEMM = 2.0 ** -23  # worst measured error / bound 0.51
# 2 to 3 layers.  Worst measured: K / V 2.08e-3 of the row rms (qwen2.5-reduced, layer 1), logits 1.89e-3 of their
# rms (qwen2.5-reduced): margins 2.4x and 2.6x.  The 12k-position case measured 1.69e-3 and 1.35e-3.
KV_TAU = 5e-3
LOGIT_TAU = 5e-3
# TinyLlama-1.1B, 22 layers.  Worst measured: K / V 7.83e-3 (layer 19; 1.4e-4 in layer 0, 1.8e-3 in layer 1, then
# slowly growing), logits 5.68e-3: margins 2.6x and 3.5x.
KV_TAU_DEEP = 2e-2
LOGIT_TAU_DEEP = 2e-2


def report(*parts):
    print("[prefill-model]", *parts, flush=True)


# ---- GEMM ---------------------------------------------------------------------------------------------------
TOKENS = [1, 31, 32, 33, 64, 65, 128, 129, 255, 256, 257, 513]  # both sides of every BN switch
ROWS = [1, 64, 127, 128, 129, 1000, 5632]  # 1, 64, 129: the CTA's second warpgroup has no row in range
K_FP32 = [4, 28, 36, 128, 160, 2048, 11008]  # tails of a 32-column K block, one ring of 4 blocks, its wrap
K_GROUP_W8 = [(32, 32), (64, 64), (128, 128), (256, 256), (256, 32), (2048, 64), (4096, 128), (11008, 256),
              (2048, 32), (4096, 64), (11008, 128)]  # K == group: one 4-byte scale per row
SENTINEL = 0x7FA5A5A5  # a NaN with a payload no kernel writes
GUARD = 256


def aligned_16_not_128(n, dtype):
    """n elements whose first one sits 16 bytes past a 128-byte boundary (TMA needs 16)."""
    size = torch.empty(0, dtype=dtype).element_size()
    buf = torch.empty(n + 256 // size, dtype=dtype, device="cuda")
    off = ((-buf.data_ptr()) % 128 + 16) // size
    view = buf[off:off + n]
    assert view.data_ptr() % 128 == 16
    return view


def with_ties(t, every):
    """Set the low 13 bits of every `every`-th element to 0x1000: exactly half-way between two TF32 values."""
    u = t.view(torch.int32).reshape(-1)
    u[::every] = (u[::every] & ~0x1FFF) | 0x1000
    return t


def guarded_out(T, N):
    """out[T, N] filled with NaN inside a buffer whose GUARD floats on both sides hold SENTINEL."""
    buf = aligned_16_not_128(T * N + 2 * GUARD, torch.int32)
    buf.fill_(SENTINEL)
    out = buf[GUARD:GUARD + T * N].view(torch.float32).view(T, N)
    out.fill_(float("nan"))
    return buf, out


def check_gemm(what, out, buf, x, w_tf32):
    sync()
    guard = torch.cat([buf[:GUARD], buf[-GUARD:]])
    assert bool((guard == SENTINEL).all()), f"{what}: a store landed outside out[T, N]"
    assert bool(torch.isfinite(out).all()), f"{what}: an element of out was not written"
    err = (out.double() - gemm_ref(x, w_tf32)).abs()
    ratio = float((err / (TAU_GEMM * np.sqrt(x.shape[1]) * gemm_abs_ref(x, w_tf32))).max())
    report(what, f"worst err / bound {ratio:.3g}")
    assert ratio <= 1.0, f"{what}: worst err / bound {ratio:.3g}"


def operand_x(T, K, g):
    x = aligned_16_not_128(T * K, torch.float32).view(T, K)
    x.normal_(0, 1, generator=g)
    return with_ties(x, 7)


def gemm_cases(i, ks):
    return [(ks[(i + j) % len(ks)], ROWS[(2 * i + 3 * j) % len(ROWS)]) for j in range(4)]


@pytest.mark.parametrize("T", TOKENS)
def test_gemm_tf32_against_the_tf32_model(kllm_lib, T):
    for K, N in gemm_cases(TOKENS.index(T), K_FP32):
        g = torch.Generator(device="cuda").manual_seed(T * 7919 + K * 31 + N)
        x = operand_x(T, K, g)
        w = aligned_16_not_128(N * K, torch.float32).view(N, K)
        w.normal_(0, 0.02, generator=g)
        with_ties(w, 5)
        buf, out = guarded_out(T, N)
        assert kllm_lib.kllm_gemm_tf32(ptr(x), ptr(w), ptr(out), T, K, N, None) == 0
        check_gemm(f"gemm_tf32 T={T} K={K} N={N}", out, buf, x, w)


@pytest.mark.parametrize("T", TOKENS)
def test_gemm_w8_tf32_against_the_tf32_model(kllm_lib, T):
    for (K, group), N in gemm_cases(TOKENS.index(T), K_GROUP_W8):
        g = torch.Generator(device="cuda").manual_seed(T * 7919 + K * 31 + N + group)
        x = operand_x(T, K, g)
        q = aligned_16_not_128(N * K, torch.int8).view(N, K)
        q.copy_(torch.randint(-127, 128, (N, K), device="cuda", generator=g, dtype=torch.int8))
        n_scales = N * K // group
        s_buf = torch.empty(n_scales + 1, device="cuda")
        scales = s_buf[1:]  # 4 bytes past the allocation: scale rows are read one float at a time
        scales.copy_(torch.empty(n_scales, device="cuda").uniform_(0.5, 2.0, generator=g) * (0.02 / 127))
        with_ties(scales, 3)  # scale * q is then a tie for every power-of-two q
        buf, out = guarded_out(T, N)
        assert kllm_lib.kllm_gemm_w8_tf32(ptr(x), ptr(q), ptr(scales), ptr(out), T, K, N, group, None) == 0
        check_gemm(f"gemm_w8_tf32 T={T} K={K} N={N} group={group}", out, buf, x, dequant_w8(q, scales, group))


def test_gemm_model_pins_the_rounding_mode():
    """The bound separates rounding from truncation: with the x operand truncated to TF32 (what the tensor core
    does to an unrounded operand) the model's own result leaves TAU_GEMM far behind on a short K."""
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.empty(33, 36, device="cuda").normal_(0, 1, generator=g)
    w = torch.empty(129, 36, device="cuda").normal_(0, 0.02, generator=g)
    xt = (x.view(torch.int32) & ~0x1FFF).view(torch.float32)
    err = (gemm_ref(tf32_rna(xt), w) - gemm_ref(x, w)).abs()
    assert float((err / (TAU_GEMM * np.sqrt(36) * gemm_abs_ref(x, w))).max()) > 100


# ---- whole prefill ------------------------------------------------------------------------------------------
from kuiperllama_b200 import FLAVOURS, SHAPES, Decoder, ModelShape, synth_weights  # noqa: E402

SEQ = 352  # = 1 + 136 + 200 + 15: room for n = 257 and for the uneven chunks to end exactly at seq_len
MODEL_SHAPES = {
    "small": replace(SHAPES["small"], seq_len=SEQ),  # GQA 3, head_size 32
    "small-hs48": replace(SHAPES["small-hs48"], seq_len=SEQ),
    "hs128": ModelShape("prefill-hs128", 512, 1376, 2, 4, 2, 2048, SEQ),  # persistent engine: V split in slices
    "small-qwen": replace(SHAPES["small-qwen"], seq_len=SEQ),  # bias, half-split RoPE, eps 1e-6
    "small-int8": replace(SHAPES["small-int8"], seq_len=SEQ),
    "small-tp-int8": replace(SHAPES["small-tp-int8"], seq_len=SEQ),
    # Qwen2.5-0.5B attention geometry (14 heads / 2 kv heads, head_size 64) at two layers
    "qwen2.5-reduced": ModelShape("qwen2.5-reduced", 896, 4864, 2, 14, 2, 4096, 16384, True, flavour="qwen2"),
}
LENGTHS = [1, 255, 256, 257]  # a single row, block tails of 255 and 1, exactly one block
CHUNKS = [1, 136, 200, 15]  # uneven calls; the last one ends exactly at seq_len
# engine name -> environment
ENGINES = {
    "graph": {"KLLM_ENGINE": "graph"},
    "persistent": {"KLLM_ENGINE": "persistent"},
    "persistent-split2": {"KLLM_ENGINE": "persistent", "KLLM_ATTN_SPLIT": "2"},
    "persistent-split8": {"KLLM_ENGINE": "persistent", "KLLM_ATTN_SPLIT": "8"},
    "persistent-fast": {"KLLM_ENGINE": "persistent", "KLLM_MODE": "fast"},  # unsplit V
}
CASES = [(key, eng) for key in ("small", "small-hs48", "small-qwen", "small-int8", "small-tp-int8")
         for eng in ("graph", "persistent", "persistent-fast")]
CASES += [("hs128", eng) for eng in ENGINES] + [("qwen2.5-reduced", "graph"), ("qwen2.5-reduced", "persistent")]

_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _free():
    yield
    _CACHE.clear()
    torch.cuda.empty_cache()


def device_sincos(lib, shape):
    """The table kllm_decoder_create writes, from the same kernel (bit-checked against the reference's)."""
    sin = torch.empty(shape.seq_len, shape.head_size, device="cuda")
    cos = torch.empty_like(sin)
    assert lib.kllm_sincos_init(shape.head_size, shape.seq_len, FLAVOURS[shape.flavour], ptr(sin), ptr(cos),
                                None) == 0
    sync()
    return sin, cos


def prompt(vocab, n, seed):
    toks = np.random.default_rng(seed).integers(0, vocab, n)
    toks[:3] = (1, 0, vocab - 1)  # the first and the last embedding row
    return [int(t) for t in toks]


def model(lib, key):
    """(shape, weights, tokens, reference over SEQ tokens with the logits of every row a call ends on)."""
    if key not in _CACHE:
        shape = MODEL_SHAPES[key]
        w = synth_weights(shape, "cuda", 77)
        toks = prompt(shape.vocab_size, SEQ, 5)
        sin, cos = device_sincos(lib, shape)
        ends = [n - 1 for n in LENGTHS] + list(np.cumsum(CHUNKS) - 1)
        _CACHE[key] = (shape, w, toks, prefill_ref(w, shape, toks, 0, sin, cos, logits_at=ends))
    return _CACHE[key]


def make_decoder(monkeypatch, shape, w, engine):
    for name in ("KLLM_ENGINE", "KLLM_MODE", "KLLM_ATTN_SPLIT"):
        monkeypatch.delenv(name, raising=False)
    for name, value in ENGINES[engine].items():
        monkeypatch.setenv(name, value)
    dec = Decoder(shape, w)
    assert dec.engine == ENGINES[engine]["KLLM_ENGINE"]
    return dec


def run_prefill(dec, toks, start_pos):
    return dec.prefill_w8(toks, start_pos) if dec.shape.group_size else dec.prefill_tf32(toks, start_pos)


def check_rows(what, dec, ref, lo, hi, ref_lo=0, kv_tau=KV_TAU):
    """K / V cache rows lo .. hi - 1 of every layer against the model's rows ref_lo .. ref_lo + hi - lo - 1."""
    k, v = dec.kv_cache()
    worst = {}
    for name, got, exp in (("K", k, ref["k"]), ("V", v, ref["v"])):
        got = torch.from_numpy(got[:, lo:hi]).cuda().double()
        exp = exp[:, ref_lo:ref_lo + hi - lo]
        rms = exp.pow(2).mean(-1, keepdim=True).sqrt()
        ratio = (got - exp).abs() / (kv_tau * rms)
        worst[name] = [round(float(r), 4) for r in ratio.amax(dim=(1, 2))]
    report(what, "K / V err / bound per layer", worst)
    for name, per_layer in worst.items():
        assert max(per_layer) <= 1.0, (what, name, per_layer)


def check_logits(what, dec, nxt, logits_ref, logit_tau=LOGIT_TAU):
    got = torch.from_numpy(dec.logits()).cuda().double()
    bound = logit_tau * float(logits_ref.pow(2).mean().sqrt())
    ratio = float((got - logits_ref).abs().max()) / bound
    top2 = torch.topk(logits_ref, 2).values
    report(what, f"logits err / bound {ratio:.4g}")
    assert ratio <= 1.0, (what, ratio)
    if float(top2[0] - top2[1]) > 2 * bound:
        assert nxt == int(torch.argmax(logits_ref)), what


@pytest.mark.parametrize("key,engine", CASES)
def test_prefill_against_the_tf32_model(kllm_lib, monkeypatch, key, engine):
    """Prompts of 1, 255, 256 and 257 positions from position 0, then the same SEQ-position prompt in calls of
    1 + 136 + 200 + 15 (the last ending exactly at seq_len for the small shapes), against one model run."""
    shape, w, toks, ref = model(kllm_lib, key)
    dec = make_decoder(monkeypatch, shape, w, engine)
    for n in LENGTHS:
        nxt = run_prefill(dec, toks[:n], 0)
        check_rows(f"{key} {engine} n={n}", dec, ref, 0, n)
        check_logits(f"{key} {engine} n={n}", dec, nxt, ref["logits_at"][n - 1])
    start = 0
    for n in CHUNKS:
        nxt = run_prefill(dec, toks[start:start + n], start)
        start += n
        check_logits(f"{key} {engine} chunks to {start}", dec, nxt, ref["logits_at"][start - 1])
    check_rows(f"{key} {engine} chunks {CHUNKS}", dec, ref, 0, start)
    dec.close()


def test_prefill_scores_past_48_kb_of_shared_memory(kllm_lib, monkeypatch):
    """Qwen2.5 geometry: positions 12200 .. 12399 in one call after a 12200-position prefill, so the attention
    scores of the last rows (12400 floats) need the opt-in beyond 48 KB.  The model starts from the cache rows the
    first call left (kv_in), so it checks the second call alone."""
    shape = MODEL_SHAPES["qwen2.5-reduced"]
    _, w, _, _ = model(kllm_lib, "qwen2.5-reduced")
    first, n = 12200, 200
    assert (first + n) * 4 > 48 * 1024
    toks = prompt(shape.vocab_size, first + n, 6)
    sin, cos = device_sincos(kllm_lib, shape)
    dec = make_decoder(monkeypatch, shape, w, "graph")
    run_prefill(dec, toks[:first], 0)
    kv_in = dec.kv_cache()
    nxt = run_prefill(dec, toks[first:], first)
    ref = prefill_ref(w, shape, toks[first:], first, sin, cos, kv_in=kv_in)
    check_rows(f"qwen2.5-reduced graph {first}+{n}", dec, ref, first, first + n)
    check_logits(f"qwen2.5-reduced graph {first}+{n}", dec, nxt, ref["logits"])
    dec.close()


def test_prefill_w8_golden_checkpoint_against_the_tf32_model(kllm_lib, monkeypatch):
    """The exporter's int8 file (dim 64 = group size: one 4-byte scale per weight row) on the graph engine, to
    seq_len in uneven calls."""
    from kuiperllama_b200.checkpoint import read_checkpoint, to_device
    shape, w = read_checkpoint(str(GOLDEN / "tiny_llama2_int8.bin"), True, "llama2")
    w = to_device(w)
    toks = [int(t) for t in np.load(GOLDEN / "tiny_llama2_int8.npz")["tokens"]]
    toks += prompt(shape.vocab_size, shape.seq_len - len(toks), 8)
    sin, cos = device_sincos(kllm_lib, shape)
    calls = [1, len(toks) - 21, 20]
    ref = prefill_ref(w, shape, toks, 0, sin, cos, logits_at=list(np.cumsum(calls) - 1))
    dec = make_decoder(monkeypatch, shape, w, "graph")
    start = 0
    for n in calls:
        nxt = run_prefill(dec, toks[start:start + n], start)
        start += n
        check_logits(f"golden int8 to {start}", dec, nxt, ref["logits_at"][start - 1])
    check_rows("golden int8", dec, ref, 0, start)
    dec.close()


def test_prefill_tinyllama_depth(kllm_lib, monkeypatch):
    """TinyLlama-1.1B (22 layers, GQA 8, head_size 64) at 300 positions: how the error grows with depth."""
    shape = SHAPES["tinyllama-1.1b"]
    w = synth_weights(shape, "cuda", 77)
    toks = prompt(shape.vocab_size, 300, 9)
    sin, cos = device_sincos(kllm_lib, shape)
    ref = prefill_ref(w, shape, toks, 0, sin, cos)
    dec = make_decoder(monkeypatch, shape, w, "persistent")
    nxt = run_prefill(dec, toks, 0)
    check_rows("tinyllama-1.1b persistent n=300", dec, ref, 0, 300, kv_tau=KV_TAU_DEEP)
    check_logits("tinyllama-1.1b persistent n=300", dec, nxt, ref["logits"], logit_tau=LOGIT_TAU_DEEP)
    dec.close()
    del w
    torch.cuda.empty_cache()


# ---- refusals -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", ["small", "small-int8"])
def test_prefill_refusals_launch_nothing(kllm_lib, monkeypatch, key):
    """Out-of-range positions, an empty prompt and token ids outside the vocabulary are refused with
    KLLM_E_INVALID before any launch: the launch count and the cache stay as they were."""
    shape, w, toks, _ = model(kllm_lib, key)
    dec = make_decoder(monkeypatch, shape, w, "graph")
    run_prefill(dec, toks[:20], 0)
    k0, v0 = dec.kv_cache()
    entry = kllm_lib.kllm_decoder_prefill_w8 if shape.group_size else kllm_lib.kllm_decoder_prefill_tf32
    V, S = shape.vocab_size, shape.seq_len

    def call(tokens, start_pos, n=None):
        arr = (ctypes.c_int32 * max(len(tokens), 1))(*tokens)
        nxt = ctypes.c_int32(-7)
        before = kllm_lib.kllm_launch_count()
        rc = entry(dec.handle, arr, len(tokens) if n is None else n, start_pos, ctypes.byref(nxt))
        assert kllm_lib.kllm_launch_count() == before
        assert nxt.value == -7
        return rc

    assert len(toks) == S
    assert call(toks[:10], S - 9) == KLLM_E_INVALID  # ends one past seq_len
    assert call(toks + [1], 0) == KLLM_E_INVALID
    assert call(toks[:1], S) == KLLM_E_INVALID
    assert call(toks[:4], 0, n=0) == KLLM_E_INVALID
    assert call(toks[:4], -1) == KLLM_E_INVALID
    for bad in (-1, V, V + 1000, -(2 ** 31)):
        assert call(toks[:5] + [bad] + toks[5:9], 0) == KLLM_E_INVALID, bad
        assert call([bad], 3) == KLLM_E_INVALID, bad
    k1, v1 = dec.kv_cache()
    assert np.array_equal(k0.view(np.uint32), k1.view(np.uint32))
    assert np.array_equal(v0.view(np.uint32), v1.view(np.uint32))
    # the first and the last id are accepted, in a prefill ending exactly at seq_len
    nxt = run_prefill(dec, [0, V - 1], S - 2)
    assert 0 <= nxt < V
    dec.close()
