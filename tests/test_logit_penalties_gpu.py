"""-m gpu: step 0 of the rule with the logit bias and the frequency and presence penalties (kllm_logit_penalties_f32,
kllm_decoder_set_frequency_presence, kllm_decoder_set_logit_bias) against the numpy mirror of
kuiperllama_b200/sampling.py on both engines and both numerics.  The expected windows are built from the ids the test
itself fed.  Ids are compared only where sampling.margin() of the adjusted logits says a last-ulp difference of the
device logf / expf cannot change them."""
import numpy as np
import pytest
import torch

from gpu_util import dev, ptr, sync
from kuiperllama_b200 import KllmError, SHAPES, check, load_library, sampling, synth_weights

pytestmark = pytest.mark.gpu

MARGIN = 1e-5
BIAS = {3: 2.0, 17: -1.5, 40: 0.75, 41: -0.0}
# (T, top_k, top_p, penalty, last_n, frequency, presence, from_pos, bias): greedy, T > 0, top-k, top-p, all of it
CONFIGS = [(0.0, 0, 1.0, 1.0, 0, 0.6, 1.5, 0, {}), (0.0, 0, 1.0, 1.0, 0, 0.0, 0.0, 0, BIAS),
           (0.8, 0, 1.0, 1.0, 0, -0.3, 0.5, 5, {}), (0.8, 40, 1.0, 1.2, 16, 0.4, 0.0, 0, BIAS),
           (0.8, 0, 0.9, 1.0, 0, 0.0, 1.5, 12, BIAS), (0.7, 20, 0.8, 1.05, 0, 0.5, 1.0, 0, {5: 1.0})]


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def kernel_step0(lib, logits, bias, rep_ids, penalty, count_ids, frequency, presence):
    d = dev(logits)
    out = torch.full_like(d, float("nan"))
    r = torch.tensor(np.asarray(rep_ids, np.int32), device="cuda")
    c = torch.tensor(np.asarray(count_ids, np.int32), device="cuda")
    bi = np.array(list(bias.keys()), np.int32)
    bv = np.array(list(bias.values()), np.float32)
    vp = lambda a: a.ctypes.data if a.size else None  # noqa: E731
    check(lib.kllm_logit_penalties_f32(ptr(d), ptr(out), logits.shape[0], vp(bi), vp(bv), len(bias), penalty,
                                       ptr(r) if len(rep_ids) else None, len(rep_ids), frequency, presence,
                                       ptr(c) if len(count_ids) else None, len(count_ids), None),
          "kllm_logit_penalties_f32")
    sync()
    return out.cpu().numpy()


def mirror(logits, bias, rep_ids, penalty, count_ids, frequency, presence):
    return sampling.penalties(logits, bias=sampling.bias_table(bias, logits.shape[0]), rep_ids=rep_ids,
                              penalty=penalty, count_ids=count_ids, frequency=frequency, presence=presence)


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_kernel_matches_the_mirror(V):
    lib = load_library()
    rng = np.random.default_rng(V)
    logits = (rng.standard_normal(V) * 4).astype(np.float32)
    logits[:6] = [0.0, -0.0, -1e-30, 3e38, -0.0, 1.0]
    hist = np.concatenate([rng.integers(0, V, V + 300), rng.integers(0, 20, 3000),
                           [-1, -7, V, V + 5, 0, 1, 2, 3, 3, 3, 4]]).astype(np.int32)
    bias = {int(i): float(b) for i, b in zip(rng.choice(V, 100, replace=False), rng.standard_normal(100) * 3)}
    bias.update({0: -0.0, 4: 0.5})
    for theta, f, p, b in [(1.0, 0.5, 1.5, bias), (1.3, 0.0, 0.0, bias), (1.05, -0.4, 1.0, {}), (0.8, 2.0, -1.0, bias),
                           (1.0, 0.0, 0.0, {})]:
        for rep, cnt in [(hist, hist), (hist[:100], hist[50:]), ([], hist), (hist, [])]:
            out = kernel_step0(lib, logits, b, rep, theta, cnt, f, p)
            assert (bits(out) == bits(mirror(logits, b, rep, theta, cnt, f, p))).all(), (V, theta, f, p, len(b))
    # only a repetition penalty: kllm_repetition_penalty_f32 bit for bit
    d = dev(logits)
    ref = torch.full_like(d, float("nan"))
    h = torch.tensor(hist, device="cuda")
    check(lib.kllm_repetition_penalty_f32(ptr(d), ptr(ref), V, ptr(h), len(hist), 1.3, None), "kllm_repetition_penalty_f32")
    sync()
    assert (bits(kernel_step0(lib, logits, {}, hist, 1.3, hist, 0.0, 0.0)) == bits(ref.cpu().numpy())).all()


def test_kernel_refusals():
    lib = load_library()
    d = dev(np.zeros(16, np.float32))
    out = torch.zeros(16, device="cuda")
    ids = torch.zeros(4, dtype=torch.int32, device="cuda")
    bi = np.array([1, 2], np.int32)
    bv = np.array([1.0, 2.0], np.float32)

    def call(logits=ptr(d), o=ptr(out), n=16, b_ids=bi.ctypes.data, b=bv.ctypes.data, nb=2, theta=1.1, rep=ptr(ids),
             nrep=4, f=0.5, p=0.5, cnt=ptr(ids), ncnt=4):
        return lib.kllm_logit_penalties_f32(logits, o, n, b_ids, b, nb, theta, rep, nrep, f, p, cnt, ncnt, None)

    assert call() == 0
    sync()
    assert call(o=ptr(d)) == -1  # in place
    assert call(logits=None) == -1 and call(o=None) == -1 and call(n=0) == -1
    assert call(b_ids=None) == -1 and call(b=None) == -1 and call(rep=None) == -1 and call(cnt=None) == -1
    assert call(nb=-1) == -1 and call(nrep=-1) == -1 and call(ncnt=-1) == -1
    for bad in (float("nan"), float("inf"), float("-inf")):
        assert call(f=bad) == -1 and call(p=bad) == -1 and call(theta=bad) == -1
    assert call(theta=0.0) == -1
    for ids_, vals in [([1, 16], [1.0, 2.0]), ([-1, 2], [1.0, 2.0]), ([2, 2], [1.0, 2.0]), ([1, 2], [1.0, np.nan]),
                       ([1, 2], [np.inf, 1.0])]:
        a, v = np.array(ids_, np.int32), np.array(vals, np.float32)
        assert call(b_ids=a.ctypes.data, b=v.ctypes.data) == -1, (ids_, vals)
    # NULL is fine where the count is 0
    assert call(b_ids=None, b=None, nb=0, rep=None, nrep=0, cnt=None, ncnt=0) == 0
    sync()


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


def configure(dec, cfg, seed):
    T, k, p, theta, last_n, f, pr, from_pos, bias = cfg
    dec.set_sampling(T, k, seed, top_p=p)
    dec.set_repetition_penalty(theta, last_n)
    dec.set_frequency_presence(f, pr, from_pos)
    dec.set_logit_bias(bias)


def expected(lg, hist, pos, cfg, seed):
    """(id, margin) of the rule at `pos` over the raw logits lg and the fed history."""
    T, k, p, theta, last_n, f, pr, from_pos, bias = cfg
    adj = mirror(lg, bias, sampling.history_window(hist, pos, last_n), theta, sampling.count_window(hist, pos, from_pos),
                 f, pr)
    return sampling.sample(adj, T, k, seed, pos, top_p=p), sampling.margin(adj, T, k, seed, pos, top_p=p)


def step_loop(dec, feed, cfg, seed, steps, start_tok=1, start_pos=0, teacher=None):
    tok, ids, checked, skipped = start_tok, [], 0, 0
    for pos in range(start_pos, start_pos + steps):
        if teacher is not None:
            tok = teacher[pos - start_pos]
        feed.put(pos, [tok])
        tok = dec.step(tok, pos)
        ids.append(tok)
        want, m = expected(dec.logits(), dec.history(), pos, cfg, seed)
        assert (dec.history() == feed.ids).all()
        if m < MARGIN:
            skipped += 1
        else:
            assert tok == want, (pos, cfg, seed)
            checked += 1
    assert skipped <= max(1, checked // 10), (checked, skipped)
    return ids


@pytest.mark.parametrize("name", ["small", "small-int8", "small-qwen"])
@pytest.mark.parametrize("numerics", ["exact", "fast"])
def test_decoder_follows_the_rule_in_every_entry(engine, name, numerics):
    dec = make(name, numerics)
    assert dec.engine == engine
    feed = Feed(dec)
    for ci, cfg in enumerate(CONFIGS):
        seed = 300 + ci
        configure(dec, cfg, seed)
        ids = step_loop(dec, feed, cfg, seed, 24)
        assert dec.generate(1, 0, 24) == ids, ("generate differs from the step loop", cfg)
        assert dec.generate_until(1, 0, 24) == ids, ("generate_until differs from the step loop", cfg)
        stop = ids[9]
        assert dec.generate_until(1, 0, 24, stop_ids=[stop]) == ids[:ids.index(stop) + 1], cfg
        teacher = [1] + [int(t) for t in np.random.default_rng(ci).integers(0, dec.shape.vocab_size, 23)]
        forced = step_loop(dec, feed, cfg, seed, 24, teacher=teacher)
        assert dec.generate(1, 0, 24, teacher=teacher) == forced, ("teacher-forced generate", cfg)
        prompt = [1] + ids[:11]
        for fn in [dec.prompt] + ([dec.prefill_w8] if SHAPES[name].group_size else [dec.prefill_tf32]):
            nxt = fn(prompt, 0)
            feed.put(0, prompt)
            assert (dec.history() == feed.ids).all()
            want, m = expected(dec.logits(), feed.ids, 11, cfg, seed)
            if m >= MARGIN:
                assert nxt == want, (fn.__name__, cfg)
    dec.close()


def run_all(monkeypatch, eng, name, cfg, seed, steps=40):
    monkeypatch.setenv("KLLM_ENGINE", eng)
    dec = make(name)
    assert dec.engine == eng
    if cfg is not None:
        configure(dec, cfg, seed)
    out = (dec.generate(1, 0, steps), dec.generate_until(2, 0, steps), dec.prompt([1, 4, 4, 9, 4], 0))
    dec.close()
    return out


@pytest.mark.parametrize("name", ["small", "small-qwen"])
def test_engines_agree(monkeypatch, name):
    for ci, cfg in enumerate(CONFIGS):
        assert run_all(monkeypatch, "persistent", name, cfg, 50 + ci) == run_all(monkeypatch, "graph", name, cfg, 50 + ci)


def test_off_settings_change_nothing(engine):
    fresh = make("small")
    base_ids = fresh.generate(1, 0, 40)
    base = (fresh.logits(), fresh.kv_cache(), fresh.history())
    fresh.close()

    def same(dec):
        assert dec.generate(1, 0, 40) == base_ids
        lg, (k, v), h = dec.logits(), dec.kv_cache(), dec.history()
        assert (bits(lg) == bits(base[0])).all() and (bits(k) == bits(base[1][0])).all()
        assert (bits(v) == bits(base[1][1])).all() and (h == base[2]).all()

    dec = make("small")
    dec.set_frequency_presence(0.0, 0.0, 3)
    dec.set_logit_bias({})
    same(dec)
    dec.set_frequency_presence(0.8, 1.5, 0)
    dec.set_logit_bias({5: 3.0})
    assert dec.generate(1, 0, 40) != base_ids, "the settings must change this greedy run"
    dec.set_frequency_presence(0.0, -0.0, 0)  # and back off
    dec.set_logit_bias(None)
    same(dec)
    dec.close()


def test_refusals_leave_the_settings(engine):
    dec = make("small")
    V = dec.shape.vocab_size
    dec.set_frequency_presence(0.5, 1.0, 2)
    dec.set_logit_bias({7: 4.0, 8: -2.0})
    want = dec.generate(1, 0, 40)
    for bad in [(float("nan"), 0.0, 0), (0.0, float("inf"), 0), (float("-inf"), 1.0, 0), (0.5, 1.0, -1)]:
        with pytest.raises(KllmError):
            dec.set_frequency_presence(*bad)
    for bad in [{V: 1.0}, {-1: 1.0}, {3: float("nan")}, {3: float("inf")}]:
        with pytest.raises(KllmError):
            dec.set_logit_bias(bad)
    lib = dec.lib
    ids = (np.array([3, 3], np.int32), np.array([1.0, 2.0], np.float32))
    assert lib.kllm_decoder_set_logit_bias(dec.handle, ids[0].ctypes.data, ids[1].ctypes.data, 2) == -1  # repeated
    assert lib.kllm_decoder_set_logit_bias(dec.handle, None, None, 2) == -1
    assert lib.kllm_decoder_set_logit_bias(dec.handle, None, None, -1) == -1
    assert dec.generate(1, 0, 40) == want, "a refusal must leave the settings in force"
    # each setter leaves the others alone
    dec.set_repetition_penalty(1.0, 0)
    dec.set_sampling(0.0, 0, 0)
    assert dec.generate(1, 0, 40) == want
    dec.close()


def test_logprobs_are_over_the_raw_logits(engine):
    tokens = [1] + [int(t) for t in np.random.default_rng(4).integers(0, 512, 30)]
    runs = []
    for cfg in [None, CONFIGS[4]]:
        dec = make("small")
        if cfg is not None:
            configure(dec, cfg, 9)
        dec.set_logprobs(5)
        dec.generate(1, 0, 30, teacher=tokens[:30])
        _, _, top_ids, top_lp = dec.logprobs(0, 30)
        runs.append((top_ids, bits(top_lp), bits(dec.score(tokens))))
        dec.close()
    assert all((a == b).all() for a, b in zip(*runs))


def test_large_biases_force_and_ban(engine):
    dec = make("small-qwen")
    dec.set_sampling(0.9, 0, 5)
    forced = 123
    dec.set_logit_bias({forced: 100.0})
    assert dec.generate(1, 0, 48) == [forced] * 48
    dec.set_logit_bias(None)
    free = dec.generate(1, 0, 48)
    top = max(set(free), key=free.count)
    dec.set_logit_bias({top: -100.0})
    assert top not in dec.generate(1, 0, 48)
    assert top not in dec.generate_until(1, 0, 48)
    dec.close()


def test_long_window_on_a_full_size_vocabulary(engine):
    """Qwen2.5-0.5B's shape over a 4 096-token context of few distinct ids: a window far longer than one CTA's
    threads, counts far above 1, and the mark words reset between tokens."""
    dec = make("qwen2.5-0.5b")
    V = dec.shape.vocab_size
    rng = np.random.default_rng(12)
    n = 4096
    prompt = [int(t) for t in rng.choice(rng.integers(0, V, 300), n)]  # 300 distinct ids, ~14 times each
    cfg = (0.0, 0, 1.0, 1.1, 0, 0.05, 0.7, 0, {int(prompt[0]): 1.0})
    configure(dec, cfg, 0)
    feed = Feed(dec)
    nxt = dec.prompt(prompt, 0)
    feed.put(0, prompt)
    want, m = expected(dec.logits(), feed.ids, n - 1, cfg, 0)
    assert m < MARGIN or nxt == want
    step_loop(dec, feed, cfg, 0, 12, start_tok=nxt, start_pos=n)
    cfg2 = (0.7, 20, 0.8, 1.0, 0, 0.3, 1.2, 2000, {})
    configure(dec, cfg2, 77)
    step_loop(dec, feed, cfg2, 77, 12, start_tok=1, start_pos=n + 12)
    dec.close()
