"""-m gpu: the wgmma prompt GEMM (kllm_gemm_tf32) -- an explicitly TOLERANCED kernel.

out[T, N] = x[T, K] . w[N, K]^T with TF32 operands (10 mantissa bits each) and fp32 accumulation in
registers.  Tolerance, stated: per element |out - exact| <= 4e-3 * sqrt(K) * rms(x row) * rms(w row).
The kernel rounds both fp32 operands to the nearest tf32 (10 mantissa bits, relative error up to 2^-11
each) before the MMA, so an element -- a sum of K such products -- is off by a few 1e-4 * sqrt(K) * rms * rms;
the bound leaves a wide margin over that."""
import ctypes

import numpy as np
import pytest
import torch

from gpu_util import ptr, sync

pytestmark = pytest.mark.gpu

SHAPES = [
    # T, K, N                      (prompt length, in_dim, out_dim)
    (1, 64, 128), (7, 288, 288), (32, 2048, 2048), (33, 2048, 256), (100, 2048, 5632),
    (128, 5632, 2048), (256, 896, 4864), (300, 2048, 2560), (17, 4096, 1000), (64, 172, 96),
]


@pytest.mark.parametrize("T,K,N", SHAPES)
def test_gemm_tf32_matches_fp64_within_tf32_tolerance(kllm_lib, T, K, N):
    g = torch.Generator(device="cuda").manual_seed(T * 131 + K * 7 + N)
    x = torch.empty(T, K, device="cuda").normal_(0, 1, generator=g)
    w = torch.empty(N, K, device="cuda").normal_(0, 0.02, generator=g)
    out = torch.full((T, N), float("nan"), device="cuda")
    assert kllm_lib.kllm_gemm_tf32(ptr(x), ptr(w), ptr(out), T, K, N, None) == 0
    sync()
    exact = (x.double() @ w.double().t())
    bound = 4e-3 * np.sqrt(K) * x.pow(2).mean(1).sqrt()[:, None] * w.pow(2).mean(1).sqrt()[None, :]
    err = (out.double() - exact).abs()
    assert torch.isfinite(out).all()
    assert bool((err <= bound.double()).all()), f"max err/bound {float((err / bound.double()).max()):.3f}"
    # and it is close in the ordinary sense
    rel = float(err.max() / exact.abs().max())
    assert rel < 4e-3, rel


def test_gemm_tf32_rejects_unaligned(kllm_lib):
    x = torch.zeros(4, 30, device="cuda"); w = torch.zeros(8, 30, device="cuda"); out = torch.zeros(4, 8, device="cuda")
    assert kllm_lib.kllm_gemm_tf32(ptr(x), ptr(w), ptr(out), 4, 30, 8, None) != 0  # in_dim % 4 != 0
    assert kllm_lib.kllm_gemm_tf32(None, ptr(w), ptr(out), 4, 32, 8, None) != 0


@pytest.mark.parametrize("engine", ["persistent", "graph"])
@pytest.mark.parametrize("key,n_prompt", [("small", 70), ("small-qwen", 40), ("tinyllama-1.1b", 300)])
def test_batched_prefill_matches_stepping_within_tf32_tolerance(kllm_lib, monkeypatch, engine, key, n_prompt):
    """kllm_decoder_prefill_tf32 (wgmma GEMMs over the whole prompt) against the bit-exact
    position-by-position prompt path on the same decoder engine.  Stated tolerance: K / V cache rows
    within 5e-2 * (row rms + 1e-3) per element (the TF32 rounding errors of every earlier layer ride
    on the residual stream), final logits within 2e-2 * max|logit| of the exact
    ones, the same greedy id when the exact top-2 margin exceeds that bound -- and decoding can go on
    from the prefilled cache (16 teacher-forced steps stay within the same logit tolerance)."""
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    monkeypatch.setenv("KLLM_ENGINE", engine)
    shape = SHAPES[key]
    w = synth_weights(shape, "cuda", 77)
    rng = np.random.default_rng(9)
    toks = [1] + [int(t) for t in rng.integers(2, shape.vocab_size, n_prompt - 1)]
    exact = Decoder(shape, w)
    nxt_e = exact.prompt(toks)
    ke, ve = exact.kv_cache(); le = exact.logits()
    fast = Decoder(shape, w)
    nxt_f = fast.prefill_tf32(toks)
    kf, vf = fast.kv_cache(); lf = fast.logits()
    n = len(toks)
    for name, a, b in (("K", ke, kf), ("V", ve, vf)):
        a, b = a[:, :n], b[:, :n]
        rms = np.sqrt((a.astype(np.float64) ** 2).mean(axis=-1, keepdims=True))
        assert np.all(np.abs(a - b) <= 5e-2 * (rms + 1e-3)), (name, float((np.abs(a - b) / (rms + 1e-3)).max()))
    tol = 2e-2 * np.abs(le).max()
    assert np.abs(le - lf).max() <= tol
    top2 = np.sort(le)[-2:]
    if top2[1] - top2[0] > 2 * tol:
        assert nxt_e == nxt_f
    # continue decoding from both caches with the same (exact) tokens
    tok = nxt_e
    for pos in range(n, n + 16):
        a = exact.step(tok, pos); b = fast.step(tok, pos)
        la, lb = exact.logits(), fast.logits()
        assert np.abs(la - lb).max() <= tol, pos
        tok = a
    exact.close(); fast.close()


def test_batched_prefill_refuses_int8(kllm_lib):
    from kuiperllama_b200 import SHAPES, Decoder, KllmError, synth_weights
    shape = SHAPES["small-int8"]
    dec = Decoder(shape, synth_weights(shape, "cuda", 3))
    with pytest.raises(KllmError):
        dec.prefill_tf32([1, 2, 3])
    assert dec.prompt([1, 2, 3]) >= 0  # the bit-exact prompt path takes every checkpoint
    dec.close()
