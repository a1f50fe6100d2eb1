"""CPU: step 0 of the sampling rule with the logit bias (0a), the repetition penalty (0b) and the frequency and
presence penalties (0c, 0d) in the numpy mirror, kuiperllama_b200/sampling.py: bit for bit against transformers'
SequenceBiasLogitsProcessor then RepetitionPenaltyLogitsProcessor, then a torch fp32 restatement of vLLM's
frequency and presence lines, and the edge cases."""
import numpy as np
import pytest

from kuiperllama_b200 import sampling


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def vllm_frequency_presence(torch, logits, counts, frequency, presence):
    """vLLM's apply_penalties lines, `logits -= frequency * output_bin_counts` and `logits -= presence *
    output_mask`, in torch fp32.  vLLM also subtracts alpha * 0 from every uncounted logit, which for a negative
    alpha turns a -0.0 logit into +0.0; the rule leaves uncounted logits alone, so the lines are applied to the
    counted ids only."""
    f = torch.tensor([[frequency]], dtype=torch.float32)
    p = torch.tensor([[presence]], dtype=torch.float32)
    mask = counts > 0
    out = logits.clone()
    out = torch.where(mask, out - f * counts, out) if frequency != 0 else out
    out = torch.where(mask, out - p * mask, out) if presence != 0 else out
    return out


def reference(logits, bias_map, rep_ids, penalty, count_ids, frequency, presence):
    transformers = pytest.importorskip("transformers")
    torch = pytest.importorskip("torch")
    V = logits.shape[0]
    x = torch.tensor(logits[None])
    if bias_map:
        proc = transformers.SequenceBiasLogitsProcessor({(int(i),): float(b) for i, b in bias_map.items()})
        x = proc(torch.zeros((1, 1), dtype=torch.long), x)
    valid_rep = np.asarray(rep_ids, np.int64)
    valid_rep = valid_rep[(valid_rep >= 0) & (valid_rep < V)]
    if penalty != 1.0 and valid_rep.size:
        x = transformers.RepetitionPenaltyLogitsProcessor(penalty)(torch.tensor(valid_rep[None]), x)
    valid = np.asarray(count_ids, np.int64)
    valid = valid[(valid >= 0) & (valid < V)]
    counts = torch.bincount(torch.tensor(valid, dtype=torch.long), minlength=V)[None]
    return vllm_frequency_presence(torch, x, counts, frequency, presence)[0].numpy()


def mirror(logits, bias_map, rep_ids, penalty, count_ids, frequency, presence):
    return sampling.penalties(logits, bias=sampling.bias_table(bias_map, logits.shape[0]), rep_ids=rep_ids,
                              penalty=penalty, count_ids=count_ids, frequency=frequency, presence=presence)


# (penalty, frequency, presence, with a bias): each part alone, all together, negative alphas
SETTINGS = [(1.0, 0.0, 0.0, True), (1.3, 0.0, 0.0, False), (1.0, 0.5, 0.0, False), (1.0, 0.0, 1.5, False),
            (1.05, 0.7, 1.5, True), (0.8, -0.4, -1.0, True), (1.0, -2.0, 2.0, False), (3.0, 0.01, 0.0, True)]


@pytest.mark.parametrize("penalty,frequency,presence,with_bias", SETTINGS)
def test_mirror_is_hf_then_vllm_bit_for_bit(penalty, frequency, presence, with_bias):
    rng = np.random.default_rng(int(penalty * 100 + frequency * 10 + presence))
    V = 32000
    logits = (rng.standard_normal(V) * 4).astype(np.float32)
    logits[:10] = [0.0, -0.0, 1e-30, -1e-30, 3e38, -3e38, 1.0, -1.0, -0.0, 0.0]
    hist = np.concatenate([rng.integers(0, V, 3000), np.arange(10), rng.integers(0, 50, 400),  # many repeats
                           [-1, -7, V, V + 3]])  # no id, and ids outside the vocabulary
    rng.shuffle(hist)
    bias_map = {}
    if with_bias:
        for i in rng.choice(V, 100, replace=False):
            bias_map[int(i)] = float(rng.standard_normal() * 5)
        bias_map.update({0: -0.0, 1: 0.0, 2: 100.0, 3: -100.0, 8: 0.25})
    for pos, last_n, from_pos in [(len(hist) - 1, 0, 0), (len(hist) - 1, 64, 1000), (2000, 500, 1500),
                                  (1000, 0, 1001)]:  # from_pos after pos: nothing counted
        rep = sampling.history_window(hist, pos, last_n)
        counted = sampling.count_window(hist, pos, from_pos)
        want = reference(logits, bias_map, rep, penalty, counted, frequency, presence)
        got = mirror(logits, bias_map, rep, penalty, counted, frequency, presence)
        assert (bits(got) == bits(want)).all(), (pos, last_n, from_pos, np.flatnonzero(bits(got) != bits(want))[:8])


def test_count_window():
    hist = np.array([10, 11, 12, 13, 14, 15, -1, -1], np.int32)
    assert sampling.count_window(hist, 5, 0).tolist() == [10, 11, 12, 13, 14, 15]
    assert sampling.count_window(hist, 5, 3).tolist() == [13, 14, 15]
    assert sampling.count_window(hist, 5, 5).tolist() == [15]
    assert sampling.count_window(hist, 5, 6).tolist() == []  # from_pos after pos: the first draw after a prompt
    assert sampling.count_window(hist, 2, 100).tolist() == []


def test_counts_and_presence_are_exact():
    lg = np.array([4.0, -4.0, 1.0, 2.0, -0.0], np.float32)
    out = sampling.frequency_presence(lg, [0, 0, 0, 1, 4, -1, 5, 99], 0.5, 0.25)
    assert out.tolist() == [4.0 - 1.5 - 0.25, -4.0 - 0.5 - 0.25, 1.0, 2.0, -0.75]
    assert (bits(sampling.frequency_presence(lg, [], 0.5, 0.25)) == bits(lg)).all()
    assert (bits(sampling.frequency_presence(lg, [0, 1, 2], 0.0, 0.0)) == bits(lg)).all()


def test_negative_alpha_raises_and_keeps_uncounted_zeros():
    lg = np.array([-0.0, 0.0, -0.0, 1.0], np.float32)
    out = sampling.frequency_presence(lg, [2, 3, 3], -1.0, -0.5)
    assert out.tolist() == [0.0, 0.0, 1.5, 3.5]
    assert np.signbit(out[0]) and not np.signbit(out[1])  # not counted: untouched, sign of zero included


def test_bias_is_skipped_without_a_map_and_adds_zero_with_one():
    lg = np.array([-0.0, 0.0, -2.5, 7.0], np.float32)
    assert sampling.bias_table({}, 4) is None
    assert (bits(sampling.apply_bias(lg, None)) == bits(lg)).all()  # -0.0 stays -0.0
    out = sampling.apply_bias(lg, sampling.bias_table({3: -1.0}, 4))
    assert out.tolist() == [0.0, 0.0, -2.5, 6.0]
    assert not np.signbit(out[0])  # -0.0 + 0 is +0.0, as HF's scores + bias
    assert not np.signbit(sampling.bias_table({1: -0.0}, 4)[1])  # HF builds the table as 0 + b


def test_order_bias_then_repetition_then_frequency_then_presence():
    lg = np.array([3.0, -3.0], np.float32)
    out = sampling.penalties(lg, bias=sampling.bias_table({0: 1.0, 1: 1.0}, 2), rep_ids=[0, 1], penalty=2.0,
                             count_ids=[0, 0, 1], frequency=0.5, presence=0.25)
    # 0: (3 + 1) / 2 - 0.5 * 2 - 0.25;  1: (-3 + 1) * 2 - 0.5 - 0.25
    assert out.tolist() == [0.75, -4.75]


def test_large_biases_force_and_ban():
    rng = np.random.default_rng(5)
    lg = (rng.standard_normal(1000) * 3).astype(np.float32)
    forced = sampling.penalties(lg, bias=sampling.bias_table({123: 100.0}, 1000))
    assert sampling.sample(forced, 0.0, 0, 0, 0) == 123
    top = int(np.argmax(lg))
    banned = sampling.penalties(lg, bias=sampling.bias_table({top: -100.0}, 1000))
    assert sampling.sample(banned, 0.0, 0, 0, 0) != top
