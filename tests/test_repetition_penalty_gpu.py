"""-m gpu: the repetition penalty, steps 0 and 0b of the rule (kllm_repetition_penalty_f32,
kllm_decoder_set_repetition_penalty, kllm_decoder_read_history), against the numpy mirror of
kuiperllama_b200/sampling.py on both engines.  The expected window is built from the ids the test itself fed, so
the device history is checked too.  Ids are compared only where sampling.margin() of the penalised logits says a
last-ulp difference of the device logf / expf cannot change them."""
import numpy as np
import pytest
import torch
from scipy import stats

from gpu_util import dev, ptr, sync
from kuiperllama_b200 import KllmError, SHAPES, check, load_library, sampling, synth_weights

pytestmark = pytest.mark.gpu

MARGIN = 1e-5
QWEN_INSTRUCT = (0.7, 20, 0.8, 1.05)  # Qwen2.5-Instruct's generation config: T, top_k, top_p, repetition_penalty
# (T, top_k, top_p, penalty, last_n): greedy, T > 0, top_k 40, top_k 300 (the whole-vector path), top-p alone,
# Qwen's full config, a boost
CONFIGS = [(0.0, 0, 1.0, 1.3, 0), (0.8, 0, 1.0, 1.2, 64), (0.8, 40, 1.0, 1.5, 1), (0.9, 300, 1.0, 1.3, 0),
           (0.8, 0, 0.9, 1.2, 64), (*QWEN_INSTRUCT, 0), (0.0, 0, 1.0, 0.8, 64)]


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def kernel_penalize(lib, logits, ids, theta):
    d = dev(logits)
    out = torch.full_like(d, float("nan"))
    di = torch.tensor(np.asarray(ids, np.int32), device="cuda")
    check(lib.kllm_repetition_penalty_f32(ptr(d), ptr(out), logits.shape[0], ptr(di) if len(ids) else None, len(ids),
                                          theta, None), "kllm_repetition_penalty_f32")
    sync()
    return out.cpu().numpy()


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_kernel_matches_the_mirror(V):
    lib = load_library()
    rng = np.random.default_rng(V)
    logits = (rng.standard_normal(V) * 4).astype(np.float32)
    logits[:4] = [0.0, -0.0, -1e-30, 3e38]
    ids = np.concatenate([rng.integers(0, V, V + 300), [-1, -7, V, V + 5, 0, 1, 2, 3, 3, 3]]).astype(np.int32)
    for theta in (1.05, 3.0, 0.8, 1.0):
        out = kernel_penalize(lib, logits, ids, theta)
        assert (bits(out) == bits(sampling.penalize(logits, ids, theta))).all(), (V, theta)
    assert (bits(kernel_penalize(lib, logits, [], 1.3)) == bits(logits)).all()


def test_kernel_refusals():
    lib = load_library()
    d = dev(np.zeros(16, np.float32))
    out = torch.zeros(16, device="cuda")
    ids = torch.zeros(4, dtype=torch.int32, device="cuda")
    for theta in (0.0, -1.0, float("nan"), float("inf"), float("-inf")):
        assert lib.kllm_repetition_penalty_f32(ptr(d), ptr(out), 16, ptr(ids), 4, theta, None) == -1, theta
    assert lib.kllm_repetition_penalty_f32(ptr(d), ptr(d), 16, ptr(ids), 4, 1.1, None) == -1  # in place
    assert lib.kllm_repetition_penalty_f32(ptr(d), ptr(out), 16, None, 4, 1.1, None) == -1
    assert lib.kllm_repetition_penalty_f32(ptr(d), ptr(out), 16, ptr(ids), -1, 1.1, None) == -1
    assert lib.kllm_repetition_penalty_f32(ptr(d), ptr(out), 0, ptr(ids), 4, 1.1, None) == -1
    assert lib.kllm_repetition_penalty_f32(None, ptr(out), 16, ptr(ids), 4, 1.1, None) == -1


def make(name, numerics="exact", seed=2024):
    from kuiperllama_b200 import Decoder
    shape = SHAPES[name]
    return Decoder(shape, synth_weights(shape, "cuda", seed), numerics=numerics)


class Feed:
    """The ids the test fed, by position (-1: none; an id outside the vocabulary holds none)."""

    def __init__(self, dec):
        self.V = dec.shape.vocab_size
        self.ids = np.full(dec.shape.seq_len, -1, np.int64)

    def put(self, pos, ids):
        for j, t in enumerate(ids):
            self.ids[pos + j] = t if 0 <= t < self.V else -1


def expected(lg, feed, pos, T, k, p, theta, last_n, seed):
    """(id, margin) of the rule at `pos` over the raw logits lg and the fed history."""
    pen = sampling.penalize(lg, sampling.history_window(feed.ids, pos, last_n), theta)
    return sampling.sample(pen, T, k, seed, pos, top_p=p), sampling.margin(pen, T, k, seed, pos, top_p=p)


def step_loop(dec, feed, cfg, seed, steps, start_tok=1, start_pos=0, teacher=None):
    """Step loop under the penalty; every id checked against the rule on dec.logits().  Returns the ids."""
    T, k, p, theta, last_n = cfg
    tok, ids, checked, skipped = start_tok, [], 0, 0
    for pos in range(start_pos, start_pos + steps):
        if teacher is not None:
            tok = teacher[pos - start_pos]
        feed.put(pos, [tok])
        tok = dec.step(tok, pos)
        ids.append(tok)
        want, m = expected(dec.logits(), feed, pos, T, k, p, theta, last_n, seed)
        if m < MARGIN:
            skipped += 1
        else:
            assert tok == want, (pos, cfg, seed)
            checked += 1
    assert skipped <= max(1, checked // 10), (checked, skipped)
    return ids


def check_history(dec, feed):
    assert (dec.history() == feed.ids).all(), np.flatnonzero(dec.history() != feed.ids)[:10]


@pytest.mark.parametrize("name", ["small", "small-int8", "small-qwen"])
@pytest.mark.parametrize("numerics", ["exact", "fast"])
def test_decoder_follows_the_rule_in_every_entry(engine, name, numerics):
    dec = make(name, numerics)
    assert dec.engine == engine
    feed = Feed(dec)
    for ci, cfg in enumerate(CONFIGS):
        T, k, p, theta, last_n = cfg
        seed = 100 + ci
        dec.set_sampling(T, k, seed, top_p=p)
        dec.set_repetition_penalty(theta, last_n)
        ids = step_loop(dec, feed, cfg, seed, 24)
        check_history(dec, feed)
        assert dec.generate(1, 0, 24) == ids, ("generate differs from the step loop", cfg)
        check_history(dec, feed)
        assert dec.generate_until(1, 0, 24) == ids, ("generate_until differs from the step loop", cfg)
        stop = ids[9]
        until = dec.generate_until(1, 0, 24, stop_ids=[stop])
        assert until == ids[:ids.index(stop) + 1], cfg
        # teacher-forced: the step loop over the same fed ids, then generate with the teacher
        teacher = [1] + [int(t) for t in np.random.default_rng(ci).integers(0, dec.shape.vocab_size, 23)]
        forced = step_loop(dec, feed, cfg, seed, 24, teacher=teacher)
        assert dec.generate(1, 0, 24, teacher=teacher) == forced, ("teacher-forced generate", cfg)
        check_history(dec, feed)
        # the id after a prompt and after a batched prefill: the rule at the last prompt position, over the
        # prompt as history
        prompt = [1] + ids[:11]
        for fn in [dec.prompt] + ([dec.prefill_w8] if SHAPES[name].group_size else [dec.prefill_tf32]):
            nxt = fn(prompt, 0)
            feed.put(0, prompt)
            check_history(dec, feed)
            want, m = expected(dec.logits(), feed, 11, T, k, p, theta, last_n, seed)
            if m >= MARGIN:
                assert nxt == want, (fn.__name__, cfg)
    dec.close()


def test_penalty_that_changes_the_top_k_set(engine):
    """theta = 3 with the largest logits of the drawn position in the history: a candidate bound taken from the
    raw logits would miss the ids that the penalty lifts into the top-k set."""
    dec = make("small")
    V = dec.shape.vocab_size
    n = 48  # prompt length; the draw is at position n - 1
    rng = np.random.default_rng(9)
    prompt = [int(t) for t in rng.integers(0, V, n)]
    for _ in range(4):  # the prompt's head converges to the top ids of the last position's logits
        dec.prompt(prompt, 0)
        top = [int(t) for t in np.argsort(dec.logits())[::-1][:n - 8]]
        prompt = top + prompt[n - 8:]
    dec.prompt(prompt, 0)
    lg = dec.logits()
    T, k, theta = 0.8, 20, 3.0
    pen = sampling.penalize(lg, prompt, theta)
    raw_top, pen_top = set(np.argsort(lg)[-k:]), set(np.argsort(pen)[-k:])
    # ids below the raw k-th largest logit enter the set: a bound from the raw maxima would not admit them
    assert len(raw_top - pen_top) >= 3, "the penalty must move part of the top-k set"
    feed = Feed(dec)
    checked = 0
    for seed in range(40):
        for cfg in [(T, k, 1.0, theta, 0), (T, k, 0.9, theta, 0), (0.0, 0, 1.0, theta, 0), (T, 0, 0.9, theta, 0)]:
            dec.set_sampling(cfg[0], cfg[1], seed, top_p=cfg[2])
            dec.set_repetition_penalty(theta, 0)
            nxt = dec.prompt(prompt, 0)
            feed.put(0, prompt)
            want, m = expected(dec.logits(), feed, n - 1, *cfg, seed)
            if m >= MARGIN:
                assert nxt == want, (seed, cfg)
                checked += 1
    assert checked >= 120
    dec.close()


def test_history_after_every_entry(engine):
    dec = make("small-int8")
    V = dec.shape.vocab_size
    feed = Feed(dec)
    check_history(dec, feed)  # a new decoder has none
    dec.set_repetition_penalty(1.2, 0)
    ids = dec.generate(5, 0, 30)
    feed.put(0, [5] + ids[:29])
    check_history(dec, feed)
    dec.step(V + 3, 30)  # outside the vocabulary: no id
    feed.put(30, [V + 3])
    check_history(dec, feed)
    dec.step(7, 31, is_prompt=True)
    feed.put(31, [7])
    check_history(dec, feed)
    # a rewind: a shorter sequence from position 0 overwrites its own positions only
    dec.prompt([9, 8, 7, 6], 0)
    feed.put(0, [9, 8, 7, 6])
    check_history(dec, feed)
    out = dec.generate_until(3, 4, 10)
    feed.put(4, [3] + out[:-1])
    check_history(dec, feed)
    dec.prefill_w8([11, 12, 13, 14, 15, 16], 2)
    feed.put(2, [11, 12, 13, 14, 15, 16])
    check_history(dec, feed)
    teacher = [20, 21, 22, 23, 24]
    dec.generate(0, 40, 5, teacher=teacher)
    feed.put(40, teacher)
    check_history(dec, feed)
    dec.close()


def test_off_settings_and_refusals(engine):
    fresh = make("small")
    base_ids = fresh.generate(1, 0, 40)
    base_lg = fresh.logits()
    fresh.close()
    dec = make("small")
    dec.set_repetition_penalty(1.0, 64)
    assert dec.generate(1, 0, 40) == base_ids
    assert (bits(dec.logits()) == bits(base_lg)).all()
    dec.set_repetition_penalty(1.4, 0)
    pen = dec.generate(1, 0, 40)
    assert pen != base_ids, "the penalty must change this greedy run"
    for bad in [(0.0, 0), (-1.0, 0), (float("nan"), 0), (float("inf"), 0), (float("-inf"), 0), (1.2, -1)]:
        with pytest.raises(KllmError):
            dec.set_repetition_penalty(*bad)
    assert dec.generate(1, 0, 40) == pen, "a refusal must leave the settings in force"
    dec.set_sampling(0.0, 0, 0)  # the sampling settings leave the penalty alone
    assert dec.generate(1, 0, 40) == pen
    dec.set_sampling(0.8, 0, 5, top_p=0.9)
    sampled = dec.generate(1, 0, 40)
    dec.set_repetition_penalty(1.4, 0)  # and setting the penalty leaves the sampling settings alone
    assert dec.generate(1, 0, 40) == sampled
    dec.set_repetition_penalty(1.0)
    dec.set_sampling(0.0, 0, 0)
    assert dec.generate(1, 0, 40) == base_ids
    assert (bits(dec.logits()) == bits(base_lg)).all()
    dec.close()


def test_distribution_through_the_whole_model():
    """4000 seeds at one position of `tiny`: chi-square against the softmax of the penalised scores."""
    dec = make("tiny")
    pos, tok = 3, 17
    dec.generate(1, 0, pos)
    dec.step(tok, pos)
    lg = dec.logits()
    top = np.argsort(lg)[::-1]
    prefix = [1, int(top[0]), int(top[2])]  # two of the most likely ids in the history
    dec.prompt(prefix + [tok], 0)
    lg = dec.logits()
    theta = 1.5
    pen = sampling.penalize(lg, prefix + [tok], theta)
    T = float(np.std(np.sort(pen.astype(np.float64))[-16:])) or 1.0
    s = (pen / np.float32(T)).astype(np.float64)
    prob = np.exp(s - s.max())
    prob /= prob.sum()
    dec.set_repetition_penalty(theta, 0)
    counts = np.zeros(lg.shape[0], np.int64)
    for seed in range(4000):
        dec.set_sampling(T, 0, seed)
        counts[dec.step(tok, pos)] += 1
    keep = prob * 4000 >= 5
    pooled = np.append(counts[keep], counts[~keep].sum())
    want = np.append(prob[keep], prob[~keep].sum()) * 4000
    assert keep.sum() >= 4
    assert stats.chisquare(pooled, want).pvalue > 1e-3
    dec.close()


@pytest.mark.parametrize("name", ["tinyllama-1.1b", "qwen2.5-0.5b"])
def test_full_size_steps_follow_the_rule(name):
    dec = make(name)
    feed = Feed(dec)
    T, k, p, theta = QWEN_INSTRUCT
    dec.set_sampling(T, k, 1234, top_p=p)
    dec.set_repetition_penalty(theta, 0)
    step_loop(dec, feed, (T, k, p, theta, 0), 1234, 256)
    dec.set_sampling(0.0, 0, 0)
    dec.set_repetition_penalty(1.3, 64)
    step_loop(dec, feed, (0.0, 0, 1.0, 1.3, 64), 0, 256, start_pos=256)
    check_history(dec, feed)
    dec.close()
