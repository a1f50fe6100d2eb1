"""-m gpu: seeded temperature / top-k sampling (kllm_sample_f32, kllm_decoder_set_sampling) against the
numpy rule of kuiperllama_b200/sampling.py, on both engines.  Ids are compared only where the two best
perturbed scores are more than MARGIN apart (relative): the device logf may differ from numpy's in the
last ulp, which can only matter below that."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from gpu_util import dev, ptr, sync
from kuiperllama_b200 import KllmError, SHAPES, check, load_library, sampling, synth_weights

pytestmark = pytest.mark.gpu

MARGIN = 1e-5


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def kernel_sample(lib, logits_dev, n, T, k, seed, pos):
    out = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    check(lib.kllm_sample_f32(ptr(logits_dev), n, T, k, seed, pos, ptr(out), None), "kllm_sample_f32")
    sync()
    return int(out.item())


CASES = [(0.0, 0, 1, 0), (0.8, 0, 7, 3), (1.0, 0, 2**40 + 5, 100), (0.8, 40, 11, 9), (1.7, 1, 3, 1),
         (0.6, 5, 99, 31), (1.0, 2000, 5, 2), (1.2, 3000, 8, 4), (1.0, -1, 13, 6)]


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_kernel_matches_the_rule(V):
    lib = load_library()
    rng = np.random.default_rng(V)
    checked = skipped = 0
    for rep in range(4):
        logits = (rng.standard_normal(V) * 3).astype(np.float32)
        if rep == 3:  # many equal logits: ties at the top-k threshold
            logits = np.round(logits * 2) / 2
        d = dev(logits)
        for T, k, seed, pos in CASES + [(0.9, V - 1, 21, 0), (0.9, V, 22, 0)]:
            want = sampling.sample(logits, T, k, seed, pos)
            if sampling.margin(logits, T, k, seed, pos) < MARGIN:
                skipped += 1
                continue
            assert kernel_sample(lib, d, V, T, k, seed, pos) == want, (V, rep, T, k, seed, pos)
            checked += 1
    assert skipped <= checked // 10, (checked, skipped)


def test_kernel_refuses_invalid_arguments():
    lib = load_library()
    d = dev(np.zeros(16, np.float32))
    out = torch.zeros(1, dtype=torch.int64, device="cuda")
    for T, n, pos in [(-0.5, 16, 0), (float("nan"), 16, 0), (float("inf"), 16, 0), (1.0, 0, 0), (1.0, 16, -1)]:
        assert lib.kllm_sample_f32(ptr(d), n, T, 0, 0, pos, ptr(out), None) == -1
    assert lib.kllm_sample_f32(None, 16, 1.0, 0, 0, 0, ptr(out), None) == -1
    assert lib.kllm_sample_f32(ptr(d), 16, 1.0, 0, 0, 0, None, None) == -1


def make(name, numerics="exact", seed=2024):
    from kuiperllama_b200 import Decoder
    shape = SHAPES[name]
    return Decoder(shape, synth_weights(shape, "cuda", seed), numerics=numerics)


def step_loop(dec, T, k, seed, steps, start_tok=1, start_pos=0, check_rule=True):
    """Sampled step loop; every id checked against the rule on dec.logits().  Returns the ids."""
    tok, ids, checked, skipped = start_tok, [], 0, 0
    for pos in range(start_pos, start_pos + steps):
        tok = dec.step(tok, pos)
        ids.append(tok)
        if check_rule:
            lg = dec.logits()
            if sampling.margin(lg, T, k, seed, pos) < MARGIN:
                skipped += 1
            else:
                assert tok == sampling.sample(lg, T, k, seed, pos), (pos, T, k, seed)
                checked += 1
    assert skipped <= max(1, checked // 10), (checked, skipped)
    return ids


@pytest.mark.parametrize("name", ["small", "small-int8", "small-qwen"])
@pytest.mark.parametrize("numerics", ["exact", "fast"])
def test_decoder_draws_by_the_rule(engine, name, numerics):
    dec = make(name, numerics)
    assert dec.engine == engine
    # k = 300 exceeds the persistent engine's grid (132 per-CTA maxima on an H100): no lower bound, the
    # candidates overflow the scratch of these small models, and the selection runs over the whole vector
    for T, k, seed in [(0.8, 0, 5), (0.8, 40, 6), (1.3, 3, 2**33 + 1), (0.9, 300, 17)]:
        dec.set_sampling(T, k, seed)
        ids = step_loop(dec, T, k, seed, 24)
        assert dec.generate(1, 0, 24) == ids, "generate differs from the step loop"
        # the id after a prompt (and after a batched prefill) is the rule at the last prompt position
        prompt = [1] + ids[:11]
        for fn in [dec.prompt] + ([dec.prefill_w8] if SHAPES[name].group_size else [dec.prefill_tf32]):
            nxt = fn(prompt, 0)
            lg = dec.logits()
            if sampling.margin(lg, T, k, seed, 11) >= MARGIN:
                assert nxt == sampling.sample(lg, T, k, seed, 11), fn.__name__
    dec.close()


def test_same_seed_same_ids_and_greedy_is_restored(engine):
    dec = make("small")
    greedy = dec.generate(1, 0, 32)
    greedy_logits = dec.logits()
    dec.set_sampling(1.0, 0, 42)
    a = dec.generate(1, 0, 32)
    b = dec.generate(1, 0, 32)
    dec.set_sampling(1.0, 0, 43)
    c = dec.generate(1, 0, 32)
    assert a == b and a != c and a != greedy
    for T, k, seed in [(0.0, 40, 42), (0.7, 1, 42)]:
        dec.set_sampling(T, k, seed)
        assert dec.generate(1, 0, 32) == greedy
        assert np.array_equal(dec.logits().view(np.uint32), greedy_logits.view(np.uint32))
    with pytest.raises(KllmError):
        dec.set_sampling(-1.0, 0, 0)
    with pytest.raises(KllmError):
        dec.set_sampling(float("nan"), 0, 0)
    dec.close()


@pytest.mark.parametrize("name", ["small", "small-qwen"])
def test_engines_draw_identical_ids(monkeypatch, name):
    ids = {}
    for eng in ("persistent", "graph"):
        monkeypatch.setenv("KLLM_ENGINE", eng)
        dec = make(name)
        dec.set_sampling(0.9, 20, 77)
        ids[eng] = dec.generate(1, 0, 40)
        dec.set_sampling(0.9, 0, 78)
        ids[eng] += dec.generate(1, 0, 40)
        dec.close()
    assert ids["persistent"] == ids["graph"]


def test_distribution_through_the_whole_model():
    """4000 seeds at one position of `tiny`: chi-square against the softmax of that position's logits."""
    dec = make("tiny")
    pos, tok = 3, 17
    dec.generate(1, 0, pos)  # fill the cache before `pos`
    dec.step(tok, pos)
    lg = dec.logits().astype(np.float64)
    k = 16
    top = np.sort(lg)[-k:]
    T = float(np.std(top)) or 1.0
    s = (lg.astype(np.float32) / np.float32(T)).astype(np.float64)
    keep = s >= np.sort(s)[-k]
    p = np.where(keep, np.exp(s - s.max()), 0.0)
    p /= p.sum()
    counts = np.zeros(lg.shape[0], np.int64)
    for seed in range(4000):
        dec.set_sampling(T, k, seed)
        counts[dec.step(tok, pos)] += 1
    assert counts[~keep].sum() == 0
    assert stats.chisquare(counts[keep], p[keep] * 4000).pvalue > 1e-3
    dec.close()


def test_full_size_tinyllama_steps_follow_the_rule():
    dec = make("tinyllama-1.1b")
    dec.set_sampling(0.8, 40, 1234)
    step_loop(dec, 0.8, 40, 1234, 256)
    dec.set_sampling(0.8, 0, 1235)
    step_loop(dec, 0.8, 0, 1235, 64, start_pos=256)
    dec.close()
