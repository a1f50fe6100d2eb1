"""-m gpu: nucleus (top-p) sampling, step 3b of the rule (kllm_sample_top_p_f32,
kllm_decoder_set_sampling_top_p) against the numpy mirror of kuiperllama_b200/sampling.py, on both engines.
Ids are compared only where sampling.margin() says a last-ulp difference of the device logf / expf cannot
change them."""
import numpy as np
import pytest
import torch
from scipy import stats

from gpu_util import dev, ptr, sync
from kuiperllama_b200 import KllmError, SHAPES, check, load_library, sampling, synth_weights

pytestmark = pytest.mark.gpu

MARGIN = 1e-5
GRAPH_CAP = 2048  # candidates in the scratch of kllm_sample_top_p_f32 and the graph engine's draw


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def kernel_sample(lib, logits_dev, n, T, k, p, seed, pos):
    out = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    check(lib.kllm_sample_top_p_f32(ptr(logits_dev), n, T, k, p, seed, pos, ptr(out), None), "kllm_sample_top_p_f32")
    sync()
    return int(out.item())


def logit_sets(V, rng):
    """(name, logits): peaked (small nucleus: the candidate path), flat (a nucleus of most of the vocabulary:
    the whole-vector path) and runs of equal logits."""
    peaked = (rng.standard_normal(V) * 3).astype(np.float32)
    flat = (rng.standard_normal(V) * 0.1).astype(np.float32)
    ties = (np.round(rng.standard_normal(V) * 4) / 2).astype(np.float32)
    return [("peaked", peaked), ("flat", flat), ("ties", ties)]


TOP_P_CASES = [(0.5, 0, 0.9, 7, 3), (0.8, 0, 0.5, 2**40 + 5, 100), (1.0, 0, 0.95, 11, 9), (0.7, 20, 0.8, 3, 1),
               (0.6, 40, 0.9, 99, 31), (1.2, 2000, 0.7, 5, 2), (1.0, 1, 0.3, 13, 6), (0.9, 0, 1e-6, 8, 4)]


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_kernel_matches_the_rule(V):
    lib = load_library()
    rng = np.random.default_rng(V + 1)
    checked = skipped = 0
    paths = set()
    for name, logits in logit_sets(V, rng):
        d = dev(logits)
        for T, k, p, seed, pos in TOP_P_CASES:
            want = sampling.sample(logits, T, k, seed, pos, top_p=p)
            if k == 0:
                paths.add(sampling.nucleus_size(logits, T, k, p) > GRAPH_CAP)
            if sampling.margin(logits, T, k, seed, pos, top_p=p) < MARGIN:
                skipped += 1
                continue
            assert kernel_sample(lib, d, V, T, k, p, seed, pos) == want, (V, name, T, k, p, seed, pos)
            checked += 1
    assert skipped <= checked // 10, (checked, skipped)
    if V > GRAPH_CAP:
        assert paths == {False, True}  # both the candidate path and the whole-vector path ran


def test_top_p_one_is_kllm_sample_f32():
    lib = load_library()
    rng = np.random.default_rng(5)
    for V in (512, 32000, 151936):
        logits = (rng.standard_normal(V) * 3).astype(np.float32)
        d = dev(logits)
        out = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        for T, k, seed, pos in [(0.0, 0, 1, 0), (0.8, 0, 7, 3), (1.0, 0, 2**40 + 5, 100), (0.8, 40, 11, 9),
                                (1.7, 1, 3, 1), (0.6, 5, 99, 31), (1.0, 2000, 5, 2), (1.2, 3000, 8, 4), (1.0, -1, 13, 6)]:
            check(lib.kllm_sample_f32(ptr(d), V, T, k, seed, pos, ptr(out), None), "kllm_sample_f32")
            sync()
            assert kernel_sample(lib, d, V, T, k, 1.0, seed, pos) == int(out.item()), (V, T, k, seed, pos)


def test_kernel_refuses_invalid_top_p():
    lib = load_library()
    d = dev(np.zeros(16, np.float32))
    out = torch.zeros(1, dtype=torch.int64, device="cuda")
    for p in (float("nan"), 0.0, -0.5, 1.0000001, float("inf")):
        assert lib.kllm_sample_top_p_f32(ptr(d), 16, 1.0, 0, p, 0, 0, ptr(out), None) == -1, p
    assert lib.kllm_sample_top_p_f32(ptr(d), 16, -1.0, 0, 0.5, 0, 0, ptr(out), None) == -1
    assert lib.kllm_sample_top_p_f32(None, 16, 1.0, 0, 0.5, 0, 0, ptr(out), None) == -1


def make(name, numerics="exact", seed=2024):
    from kuiperllama_b200 import Decoder
    shape = SHAPES[name]
    return Decoder(shape, synth_weights(shape, "cuda", seed), numerics=numerics)


def step_loop(dec, T, k, p, seed, steps, start_tok=1, start_pos=0):
    """Sampled step loop; every id checked against the rule on dec.logits().  Returns the ids."""
    tok, ids, checked, skipped = start_tok, [], 0, 0
    for pos in range(start_pos, start_pos + steps):
        tok = dec.step(tok, pos)
        ids.append(tok)
        lg = dec.logits()
        if sampling.margin(lg, T, k, seed, pos, top_p=p) < MARGIN:
            skipped += 1
        else:
            assert tok == sampling.sample(lg, T, k, seed, pos, top_p=p), (pos, T, k, p, seed)
            checked += 1
    assert skipped <= max(1, checked // 10), (checked, skipped)
    return ids


@pytest.mark.parametrize("name", ["small", "small-int8", "small-qwen"])
@pytest.mark.parametrize("numerics", ["exact", "fast"])
def test_decoder_draws_by_the_rule(engine, name, numerics):
    dec = make(name, numerics)
    assert dec.engine == engine
    for T, k, p, seed in [(0.8, 0, 0.9, 5), (0.7, 20, 0.8, 6), (1.3, 0, 0.5, 2**33 + 1), (0.9, 300, 0.95, 17)]:
        dec.set_sampling(T, k, seed, top_p=p)
        ids = step_loop(dec, T, k, p, seed, 24)
        assert dec.generate(1, 0, 24) == ids, "generate differs from the step loop"
        assert dec.generate_until(1, 0, 24) == ids, "generate_until differs from the step loop"
        # the id after a prompt (and after a batched prefill) is the rule at the last prompt position
        prompt = [1] + ids[:11]
        for fn in [dec.prompt] + ([dec.prefill_w8] if SHAPES[name].group_size else [dec.prefill_tf32]):
            nxt = fn(prompt, 0)
            lg = dec.logits()
            if sampling.margin(lg, T, k, seed, 11, top_p=p) >= MARGIN:
                assert nxt == sampling.sample(lg, T, k, seed, 11, top_p=p), fn.__name__
    dec.close()


def test_engines_and_draw_paths_give_identical_ids(monkeypatch):
    """A temperature whose nucleus is a few tokens (candidates in shared memory) and one whose nucleus
    exceeds every engine's scratch (the selection over the whole vector), on `small` (vocabulary 4096)."""
    dec = make("small")
    dec.step(1, 0)
    lg = dec.logits()
    dec.close()
    p = 0.9
    temps = {}
    for T in (0.001, 0.002, 0.005, 0.01, 0.02, 0.05, 0.1, 0.2, 0.4, 0.8, 1.6, 3.2, 6.4, 12.8):
        size = sampling.nucleus_size(lg, T, 0, p)
        if size <= 16:
            temps.setdefault("candidates", T)
        if size > GRAPH_CAP:
            temps.setdefault("whole", T)
    assert set(temps) == {"candidates", "whole"}, temps
    ids = {}
    for eng in ("persistent", "graph"):
        monkeypatch.setenv("KLLM_ENGINE", eng)
        dec = make("small")
        for path, T in temps.items():
            dec.set_sampling(T, 0, 77, top_p=p)
            ids[eng, path] = step_loop(dec, T, 0, p, 77, 32)
        dec.set_sampling(temps["whole"], 50, 78, top_p=p)  # top-k first, then the nucleus of its candidates
        ids[eng, "top-k"] = dec.generate(1, 0, 32)
        dec.close()
    for key in ("candidates", "whole", "top-k"):
        assert ids["persistent", key] == ids["graph", key], key


def test_refusals_leave_the_settings_and_set_sampling_resets_top_p(engine):
    dec = make("small")
    dec.set_sampling(0.9, 0, 42, top_p=0.7)
    a = dec.generate(1, 0, 32)
    for bad in (float("nan"), 0.0, -0.1, 1.5):
        with pytest.raises(KllmError):
            dec.set_sampling(0.9, 0, 43, top_p=bad)
    with pytest.raises(KllmError):
        dec.set_sampling(-1.0, 0, 43, top_p=0.5)
    assert dec.generate(1, 0, 32) == a
    dec.set_sampling(0.9, 0, 42)  # top_p back to 1
    plain = dec.generate(1, 0, 32)
    fresh = make("small")
    fresh.set_sampling(0.9, 0, 42)
    assert plain == fresh.generate(1, 0, 32)
    fresh.set_sampling(0.9, 0, 42, top_p=0.7)
    assert fresh.generate(1, 0, 32) == a
    fresh.close()
    # top_p = 1 through the top-p entry is kllm_decoder_set_sampling
    check(dec.lib.kllm_decoder_set_sampling_top_p(dec.handle, 0.9, 0, 1.0, 42), "kllm_decoder_set_sampling_top_p")
    assert dec.generate(1, 0, 32) == plain
    dec.close()


def test_distribution_through_the_whole_model():
    """4000 seeds at one position of `tiny`: chi-square against the softmax renormalised over the nucleus."""
    dec = make("tiny")
    pos, tok = 3, 17
    dec.generate(1, 0, pos)  # fill the cache before `pos`
    dec.step(tok, pos)
    lg = dec.logits()
    top = np.sort(lg.astype(np.float64))[-16:]
    T = float(np.std(top)) or 1.0
    p = 0.7
    s = (lg / np.float32(T)).astype(np.float64)
    keep = sampling._keep(lg / np.float32(T), 0, p)
    assert 2 < keep.sum() < 64, keep.sum()
    prob = np.where(keep, np.exp(s - s.max()), 0.0)
    prob /= prob.sum()
    counts = np.zeros(lg.shape[0], np.int64)
    for seed in range(4000):
        dec.set_sampling(T, 0, seed, top_p=p)
        counts[dec.step(tok, pos)] += 1
    assert counts[~keep].sum() == 0
    assert stats.chisquare(counts[keep], prob[keep] * 4000).pvalue > 1e-3
    dec.close()


@pytest.mark.parametrize("name", ["tinyllama-1.1b", "qwen2.5-0.5b"])
def test_full_size_steps_follow_the_rule(name):
    dec = make(name)
    dec.set_sampling(0.7, 20, 1234, top_p=0.8)  # Qwen2.5-Instruct's generation config
    step_loop(dec, 0.7, 20, 0.8, 1234, 256)
    dec.set_sampling(0.6, 0, 1235, top_p=0.9)  # Llama-2-chat's
    step_loop(dec, 0.6, 0, 0.9, 1235, 256, start_pos=256)
    dec.close()
