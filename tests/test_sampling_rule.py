"""The numpy mirror of the sampling rule (kuiperllama_b200/sampling.py): Philox known answers, the
distribution it draws, and its top-k set.  CPU only."""
import numpy as np
import pytest
from scipy import stats

from kuiperllama_b200 import sampling


@pytest.mark.parametrize("ctr,key,out", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, out):
    assert tuple(int(x) for x in sampling.philox4x32_10(np.array(ctr, np.uint64), key)) == out


def test_uniform_rounds_toward_zero_and_stays_inside_the_unit_interval():
    k = np.array([0, (1 << 23) - 1, 1 << 23, (1 << 24) - 1], np.int64)
    x = (k << 8 | 0xFF).astype(np.uint32)  # the low 8 bits of a word do not matter
    u = sampling.uniform(x)
    assert u.dtype == np.float32
    assert list(u.astype(np.float64)) == [0.5 * 2.0 ** -24, ((1 << 23) - 0.5) * 2.0 ** -24,  # exact below 2^23
                                          0.5, 1 - 2.0 ** -24]  # truncated from k + 0.5 above
    assert (u > 0).all() and (u < 1).all()
    g = sampling.gumbel(x)
    assert np.isfinite(g).all() and g[0] < g[1] < g[2] < g[3]
    assert np.isfinite(sampling.gumbel_noise(4096, 7, 3)).all()


def _draws(logits, T, k, n_seeds, pos=5):
    return np.array([sampling.sample(logits, T, k, seed, pos) for seed in range(n_seeds)])


def _chi2(ids, probs):
    kept = np.flatnonzero(probs > 0)
    counts = np.bincount(ids, minlength=probs.shape[0])
    assert counts[probs == 0].sum() == 0, "an id outside the kept set was drawn"
    return stats.chisquare(counts[kept], probs[kept] * ids.shape[0]).pvalue


@pytest.mark.parametrize("T,k", [(1.0, 0), (0.7, 0), (1.3, 5)])
def test_draws_follow_the_softmax_of_the_kept_set(T, k):
    rng = np.random.default_rng(11)
    logits = (rng.standard_normal(12) * 1.5).astype(np.float32)
    s = (logits / np.float32(T)).astype(np.float64)
    keep = np.ones_like(s, bool) if k == 0 else s >= np.sort(s)[-k]
    p = np.where(keep, np.exp(s - s.max()), 0.0)
    p /= p.sum()
    ids = _draws(logits, T, k, 20000)
    assert _chi2(ids, p) > 1e-3


def test_ties_at_the_threshold_are_kept():
    logits = np.array([3.0, 1.0, 2.0, 2.0, 2.0, -1.0, 0.5], np.float32)  # k = 2: tau = 2.0, kept {0, 2, 3, 4}
    ids = _draws(logits, 1.0, 2, 20000)
    p = np.array([np.e, 0, 1, 1, 1, 0, 0])
    p /= p.sum()
    assert set(np.unique(ids)) == {0, 2, 3, 4}
    assert _chi2(ids, p) > 1e-3


@pytest.mark.parametrize("T", [0.1, 0.8, 1.0, 5.0])
def test_top_k_one_is_greedy(T):
    rng = np.random.default_rng(3)
    for seed in range(50):
        logits = rng.standard_normal(1000).astype(np.float32)
        assert sampling.sample(logits, T, 1, seed, seed) == int(np.argmax(logits))


def test_temperature_zero_is_greedy_and_seed_matters():
    rng = np.random.default_rng(5)
    logits = rng.standard_normal(32000).astype(np.float32)
    assert sampling.sample(logits, 0.0, 40, 9, 1) == int(np.argmax(logits))
    ids = {sampling.sample(logits, 1.0, 0, seed, 1) for seed in range(20)}
    assert len(ids) > 10
    assert sampling.sample(logits, 1.0, 0, 4, 1) == sampling.sample(logits, 1.0, 0, 4, 1)
