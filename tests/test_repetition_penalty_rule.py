"""CPU: steps 0 and 0b of the sampling rule (history window and repetition penalty) in the numpy mirror,
kuiperllama_b200/sampling.py: bit for bit against transformers' RepetitionPenaltyLogitsProcessor, the chain
penalty -> temperature -> top-k -> top-p against HF's warpers in that order, and the edge cases."""
import numpy as np
import pytest

from kuiperllama_b200 import sampling


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("theta", [1.05, 1.3, 0.8, 3.0])
def test_penalize_is_hf_bit_for_bit(theta):
    transformers = pytest.importorskip("transformers")
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(int(theta * 100))
    V = 32000
    logits = (rng.standard_normal(V) * 4).astype(np.float32)
    logits[:8] = [0.0, -0.0, 1e-30, -1e-30, 3e38, -3e38, 1.0, -1.0]
    ids = np.concatenate([rng.integers(0, V, 3000), np.arange(8), rng.integers(0, V, 50)])  # duplicates
    hf = transformers.RepetitionPenaltyLogitsProcessor(theta)(torch.tensor(ids[None]), torch.tensor(logits[None]))
    assert (bits(sampling.penalize(logits, ids, theta)) == bits(hf[0].numpy())).all()


@pytest.mark.parametrize("T,k,p,theta", [(0.7, 20, 0.8, 1.05), (1.0, 40, 1.0, 1.3), (0.9, 0, 0.9, 1.2),
                                         (1.3, 300, 0.95, 0.8), (0.5, 5, 0.5, 3.0)])
def test_chain_matches_hf_warpers(T, k, p, theta):
    """penalty -> temperature -> top-k -> top-p (transformers' _get_logits_processor order): the mirror's kept
    set, and its scores bit for bit, against HF's masked scores.  HF's nucleus is an fp32 cumsum: positions whose
    nucleus boundary is closer than 1e-5 of the mass are left out, and there must be few."""
    transformers = pytest.importorskip("transformers")
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(int(T * 1000) + k)
    V = 4096
    checked = skipped = 0
    for trial in range(20):
        logits = (rng.standard_normal(V) * 3).astype(np.float32)
        hist = rng.integers(0, V, 200)
        hist[:10] = np.argsort(logits)[-10:]  # the largest logits in the history: the penalty moves the top set
        procs = [transformers.RepetitionPenaltyLogitsProcessor(theta), transformers.TemperatureLogitsWarper(T)]
        if k > 0:
            procs.append(transformers.TopKLogitsWarper(k))
        if p < 1:
            procs.append(transformers.TopPLogitsWarper(p))
        x = torch.tensor(logits[None])
        for proc in procs:
            x = proc(torch.tensor(hist[None]), x)
        hf = x[0].numpy()
        pen = sampling.penalize(logits, hist, theta)
        s = pen / np.float32(T)
        if sampling.nucleus_margin(pen, T, k, p) < 1e-5:
            skipped += 1
            continue
        keep = sampling._keep(s, k, p)
        assert (np.isfinite(hf) == keep).all(), trial
        assert (bits(hf[keep]) == bits(s[keep])).all(), trial
        checked += 1
    assert skipped <= checked // 10, (checked, skipped)


def test_negative_zero_and_minus_zero():
    lg = np.array([-2.0, 0.0, -0.0, 3.0, -5.5, 7.25], np.float32)
    out = sampling.penalize(lg, [0, 1, 2, 3, 4], 1.5)
    th = np.float32(1.5)
    want = np.array([lg[0] * th, lg[1] / th, lg[2] / th, lg[3] / th, lg[4] * th, lg[5]], np.float32)
    assert (bits(out) == bits(want)).all()
    assert np.signbit(out[2]) and not np.signbit(out[1])  # -0.0 is not < 0: divided, and stays -0.0
    assert out[5] == lg[5]  # not in the history


def test_duplicates_are_penalised_once():
    lg = np.array([4.0, -4.0, 1.0], np.float32)
    once = sampling.penalize(lg, [0, 1], 2.0)
    assert (bits(sampling.penalize(lg, [0, 0, 0, 1, 1, 0], 2.0)) == bits(once)).all()
    assert once.tolist() == [2.0, -8.0, 1.0]


def test_theta_below_one_is_a_boost():
    lg = np.array([4.0, -4.0, 1.0], np.float32)
    out = sampling.penalize(lg, [0, 1], 0.5)
    assert out.tolist() == [8.0, -2.0, 1.0]
    assert sampling.sample(out, 0.0, 0, 0, 0) == 0


def test_theta_one_changes_nothing():
    lg = np.random.default_rng(3).standard_normal(1000).astype(np.float32)
    assert (bits(sampling.penalize(lg, np.arange(1000), 1.0)) == bits(lg)).all()


def test_history_window():
    hist = np.array([10, 11, 12, 13, 14, 15, -1, -1], np.int32)
    assert sampling.history_window(hist, 5, 0).tolist() == [10, 11, 12, 13, 14, 15]  # the whole sequence
    assert sampling.history_window(hist, 5, 1).tolist() == [15]  # only the position being drawn
    assert sampling.history_window(hist, 5, 6).tolist() == [10, 11, 12, 13, 14, 15]  # exactly pos + 1
    assert sampling.history_window(hist, 5, 100).tolist() == [10, 11, 12, 13, 14, 15]  # larger
    assert sampling.history_window(hist, 5, 3).tolist() == [13, 14, 15]
    assert sampling.history_window(hist, 0, 0).tolist() == [10]
    # the window never reaches above pos: a rewind needs no reset
    assert sampling.history_window(hist, 2, 0).tolist() == [10, 11, 12]


def test_entries_without_an_id_are_ignored():
    lg = np.array([4.0, -4.0, 1.0, 2.0], np.float32)
    out = sampling.penalize(lg, [-1, -1, 2, 4, 1000, -7], 2.0)  # -1: no id; >= V: outside the vocabulary
    assert out.tolist() == [4.0, -4.0, 0.5, 2.0]
    assert (bits(sampling.penalize(lg, [], 2.0)) == bits(lg)).all()


def test_the_penalty_comes_before_the_temperature():
    """s_i = l'_i / T: two roundings, as HF does it, not one division by theta * T."""
    rng = np.random.default_rng(11)
    lg = (rng.standard_normal(50000) * 3).astype(np.float32)
    theta, T = np.float32(1.05), np.float32(0.7)
    s = sampling.penalize(lg, np.arange(50000), theta) / T
    two = np.where(lg < 0, lg * theta, lg / theta) / T
    assert (bits(s) == bits(two)).all()
