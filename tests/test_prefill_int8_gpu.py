"""-m gpu: batched prefill of int8 checkpoints (kllm_gemm_w8_tf32, kllm_decoder_prefill_w8) -- TOLERANCED.

The int8 GEMM dequantises each weight tile in shared memory (scale * q in fp32, rounded to the nearest tf32)
and multiplies on the fp32 GEMM's wgmma tf32 path, so it keeps that GEMM's stated bound
(tests/test_prefill_gpu.py): per element |out - exact| <= 4e-3 * sqrt(K) * rms(x row) * rms(dequantised w row),
exact being the fp64 product with the dequantised weight s (.) w.  The prefill keeps the fp32 prefill's bounds:
K / V cache rows within 5e-2 * (row rms + 1e-3), last logits within 2e-2 * max|logit| of the bit-exact
position-by-position path, the same greedy id where the exact top-2 margin exceeds twice that, and 16
teacher-forced steps from the prefilled cache within the same logit bound."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN
from gpu_util import ptr, sync

pytestmark = pytest.mark.gpu

KLLM_E_INVALID, KLLM_E_UNSUPPORTED = -1, -2

GEMM_SHAPES = [
    # T, K, N       (prompt rows, in_dim, out_dim): T and N off the tile, a 4-byte scale row (K = 64), 7B shapes
    (1, 64, 64), (7, 128, 384), (33, 256, 768), (100, 4096, 4096), (256, 4096, 11008), (300, 11008, 4096),
    (17, 4096, 1000),
]


def quantized(N, K, g, group=64):
    from kuiperllama_b200.decoder import quantize_q80
    w = torch.empty(N, K, device="cuda").normal_(0, 0.02, generator=g)
    q, s = quantize_q80(w, group)
    deq = (q.double().reshape(-1, group) * s.double()[:, None]).reshape(N, K)
    return q.contiguous(), s.contiguous(), deq


@pytest.mark.parametrize("T,K,N", GEMM_SHAPES)
def test_gemm_w8_tf32_matches_fp64_within_tf32_tolerance(kllm_lib, T, K, N):
    g = torch.Generator(device="cuda").manual_seed(T * 131 + K * 7 + N)
    x = torch.empty(T, K, device="cuda").normal_(0, 1, generator=g)
    q, s, deq = quantized(N, K, g)
    out = torch.full((T, N), float("nan"), device="cuda")
    assert kllm_lib.kllm_gemm_w8_tf32(ptr(x), ptr(q), ptr(s), ptr(out), T, K, N, 64, None) == 0
    sync()
    exact = x.double() @ deq.t()
    bound = 4e-3 * np.sqrt(K) * x.double().pow(2).mean(1).sqrt()[:, None] * deq.pow(2).mean(1).sqrt()[None, :]
    err = (out.double() - exact).abs()
    assert torch.isfinite(out).all()
    assert bool((err <= bound).all()), f"max err/bound {float((err / bound).max()):.3f}"


def test_gemm_w8_tf32_refusals(kllm_lib):
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.zeros(4, 256, device="cuda")
    q, s, _ = quantized(64, 256, g)
    out = torch.zeros(4, 64, device="cuda")
    f = kllm_lib.kllm_gemm_w8_tf32
    assert f(ptr(x), ptr(q), ptr(s), ptr(out), 4, 40, 64, 40, None) == KLLM_E_UNSUPPORTED  # in_dim % 16
    assert f(ptr(x), ptr(q), ptr(s), ptr(out), 4, 96, 64, 64, None) == KLLM_E_UNSUPPORTED  # in_dim % group_size
    assert f(ptr(x), ptr(q), ptr(s), ptr(out), 4, 96, 64, 48, None) == KLLM_E_UNSUPPORTED  # group_size % 32
    for args in ((None, ptr(q), ptr(s), ptr(out)), (ptr(x), None, ptr(s), ptr(out)),
                 (ptr(x), ptr(q), None, ptr(out)), (ptr(x), ptr(q), ptr(s), None)):
        assert f(*args, 4, 256, 64, 64, None) == KLLM_E_INVALID
    assert f(ptr(x), ptr(q), ptr(s), ptr(out), 0, 256, 64, 64, None) == KLLM_E_INVALID
    assert f(ptr(x), ptr(q), ptr(s), ptr(out), 4, 256, 64, 0, None) == KLLM_E_INVALID


_WEIGHTS = {}


@pytest.fixture(scope="module", autouse=True)
def _free_weights():
    yield
    _WEIGHTS.clear()
    torch.cuda.empty_cache()


def weights(key):
    """Synthetic weights per shape, made once per module (the 7B ones take a while)."""
    from kuiperllama_b200 import SHAPES, synth_weights
    if key not in _WEIGHTS:
        _WEIGHTS[key] = synth_weights(SHAPES[key], "cuda", 77)
    return _WEIGHTS[key]


def prompt_tokens(vocab, n, seed=9):
    rng = np.random.default_rng(seed)
    return [1] + [int(t) for t in rng.integers(2, vocab, n - 1)]


def assert_within_prefill_tolerance(exact, fast, nxt_e, nxt_f, n, steps=16):
    """The stated bounds (module docstring) between a decoder that ran the exact prompt path and one that ran
    the batched prefill over the same n positions; then `steps` teacher-forced steps on both."""
    ke, ve = exact.kv_cache(); le = exact.logits()
    kf, vf = fast.kv_cache(); lf = fast.logits()
    for name, a, b in (("K", ke, kf), ("V", ve, vf)):
        a, b = a[:, :n], b[:, :n]
        rms = np.sqrt((a.astype(np.float64) ** 2).mean(axis=-1, keepdims=True))
        ratio = np.abs(a - b) / (5e-2 * (rms + 1e-3))
        per_layer = [round(float(r.max()), 4) for r in ratio]  # error growth with depth, in units of the bound
        assert np.all(ratio <= 1), (name, "max err / bound per layer", per_layer)
    tol = 2e-2 * np.abs(le).max()
    assert np.abs(le - lf).max() <= tol, float(np.abs(le - lf).max() / tol)
    top2 = np.sort(le)[-2:]
    if top2[1] - top2[0] > 2 * tol:
        assert nxt_e == nxt_f
    tok = nxt_e
    for pos in range(n, n + steps):
        a = exact.step(tok, pos); fast.step(tok, pos)
        assert np.abs(exact.logits() - fast.logits()).max() <= tol, pos
        tok = a


ENGINES = {"persistent": ("persistent", None), "persistent-fast": ("persistent", "fast"), "graph": ("graph", None)}


@pytest.mark.parametrize("engine", sorted(ENGINES))
@pytest.mark.parametrize("key,n_prompt", [("small-int8", 70), ("small-tp-int8", 40), ("llama2-7b-int8", 300)])
def test_prefill_w8_matches_exact_stepping_within_tf32_tolerance(kllm_lib, monkeypatch, engine, key, n_prompt):
    """kllm_decoder_prefill_w8 against the bit-exact prompt path (exact numerics) on the same engine.  300
    positions of the 7B shape cross a 256-position block, and its head_size 128 gives the persistent engine's
    split V layout; KLLM_MODE=fast gives that engine's unsplit one."""
    from kuiperllama_b200 import SHAPES, Decoder
    eng, mode = ENGINES[engine]
    monkeypatch.setenv("KLLM_ENGINE", eng)
    monkeypatch.delenv("KLLM_MODE", raising=False)
    shape = SHAPES[key]
    w = weights(key)
    toks = prompt_tokens(shape.vocab_size, n_prompt)
    exact = Decoder(shape, w)
    nxt_e = exact.prompt(toks)
    if mode:
        monkeypatch.setenv("KLLM_MODE", mode)
    fast = Decoder(shape, w)
    assert fast.engine == eng
    nxt_f = fast.prefill_w8(toks)
    assert_within_prefill_tolerance(exact, fast, nxt_e, nxt_f, len(toks))
    exact.close(); fast.close()


def test_prefill_w8_golden_checkpoint(kllm_lib, monkeypatch):
    """The exporter's own int8 file (dim 64: one 4-byte scale per weight row) on the graph engine."""
    from kuiperllama_b200 import Decoder
    from kuiperllama_b200.checkpoint import read_checkpoint, to_device
    monkeypatch.setenv("KLLM_ENGINE", "graph")
    shape, w = read_checkpoint(str(GOLDEN / "tiny_llama2_int8.bin"), True, "llama2")
    w = to_device(w)
    toks = [int(t) for t in np.load(GOLDEN / "tiny_llama2_int8.npz")["tokens"]]
    exact = Decoder(shape, w)
    nxt_e = exact.prompt(toks)
    fast = Decoder(shape, w)
    nxt_f = fast.prefill_w8(toks)
    assert_within_prefill_tolerance(exact, fast, nxt_e, nxt_f, len(toks), steps=min(16, shape.seq_len - len(toks)))
    exact.close(); fast.close()


def test_prefill_w8_in_two_calls_agrees_with_one(kllm_lib):
    """A prompt prefilled as [0, 137) and then [137, n) from start_pos 137 (each call its own 256-position
    blocks) against one call over [0, n)."""
    from kuiperllama_b200 import Decoder, ModelShape, synth_weights
    shape = ModelShape("prefill-int8", 256, 768, 2, 4, 2, 1024, 320, group_size=64)
    w = synth_weights(shape, "cuda", 31)
    toks = prompt_tokens(shape.vocab_size, 300, seed=4)
    one = Decoder(shape, w)
    nxt_1 = one.prefill_w8(toks)
    two = Decoder(shape, w)
    two.prefill_w8(toks[:137])
    nxt_2 = two.prefill_w8(toks[137:], start_pos=137)
    assert_within_prefill_tolerance(one, two, nxt_1, nxt_2, len(toks))
    one.close(); two.close()


def test_prefill_w8_is_deterministic(kllm_lib):
    from kuiperllama_b200 import SHAPES, Decoder
    shape = SHAPES["small-int8"]
    w = weights("small-int8")
    toks = prompt_tokens(shape.vocab_size, 70)
    outs = []
    for _ in range(2):
        dec = Decoder(shape, w)
        nxt = dec.prefill_w8(toks)
        k, v = dec.kv_cache()
        outs.append((nxt, k, v, dec.logits()))
        dec.close()
    (n0, k0, v0, l0), (n1, k1, v1, l1) = outs
    assert n0 == n1
    for a, b in ((k0, k1), (v0, v1), (l0, l1)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_prefill_w8_refuses_fp32_checkpoints(kllm_lib):
    from kuiperllama_b200 import SHAPES, Decoder, KllmError, synth_weights
    shape = SHAPES["small"]
    dec = Decoder(shape, synth_weights(shape, "cuda", 3))
    with pytest.raises(KllmError):
        dec.prefill_w8([1, 2, 3])
    assert dec.prompt([1, 2, 3]) >= 0
    dec.close()
    shape8 = SHAPES["small-int8"]
    dec8 = Decoder(shape8, weights("small-int8"))
    with pytest.raises(KllmError):
        dec8.prefill_tf32([1, 2, 3])
    assert dec8.prompt([1, 2, 3]) >= 0
    dec8.close()
