"""CPU: step 3b of the sampling rule (nucleus / top-p) in the numpy mirror, kuiperllama_b200/sampling.py,
against an independent fp64 sort-and-cumsum form of "keep a token iff the probability mass strictly above
it is below p", and its edge cases."""
import numpy as np
import pytest
from scipy import stats

from kuiperllama_b200 import sampling


def ref_keep(logits, T, k, p):
    """fp64: scores as the rule's fp32 l / T, top-k, then softmax over the kept set sorted descending; a
    token stays iff the mass of strictly larger scores is below p24 / 2^24.  Returns (keep, boundary): the
    tokens whose decision is too close to call against the rule's integer masses."""
    s = (np.asarray(logits, np.float32) / np.float32(T)).astype(np.float64)
    n = s.shape[0]
    keep = np.ones(n, bool)
    if 0 < k < n:
        keep = s >= np.sort(s)[::-1][k - 1]
    idx = np.flatnonzero(keep)
    order = idx[np.argsort(-s[idx], kind="stable")]
    sv = s[order]
    prob = np.exp(sv - sv[0])
    z = prob.sum()
    prob /= z
    excl = np.cumsum(prob) - prob
    first = np.searchsorted(-sv, -sv, side="left")  # the first of each run of equal scores
    above = excl[first]
    p_eff = max(1.0, float(np.rint(np.float64(np.float32(p)) * 2.0 ** 24))) / 2.0 ** 24
    out = np.zeros(n, bool)
    out[order] = above < p_eff
    # fp32 weights (a few ulp apart from fp64), floored to 2^-32 of the maximum: at most this much of Z
    tol = 1e-6 + n * 2.0 ** -32 / z
    boundary = np.zeros(n, bool)
    boundary[order] = np.abs(above - p_eff) < tol
    return out, boundary


def kept(logits, T, k, p):
    s = np.asarray(logits, np.float32) / np.float32(T)
    return sampling._keep(s, k, p)


@pytest.mark.parametrize("V", [12, 1000, 32000, 151936])
def test_mirror_matches_sort_and_cumsum(V):
    rng = np.random.default_rng(V)
    boundary_cases = 0
    for rep in range(3):
        logits = (rng.standard_normal(V) * (3.0 if rep < 2 else 0.3)).astype(np.float32)
        if rep == 1:
            logits = np.round(logits * 4) / 4  # runs of equal scores
        for T in (0.5, 0.8, 1.5):
            for k in (0, 40, 1000):
                for p in (0.1, 0.5, 0.9, 0.99):
                    want, boundary = ref_keep(logits, T, k, p)
                    got = kept(logits, T, k, p)
                    differ = got != want
                    # the sets agree except at tokens on the boundary itself
                    assert not (differ & ~boundary).any(), (V, rep, T, k, p, got.sum(), want.sum())
                    boundary_cases += bool(differ.any())
    assert boundary_cases <= 3, boundary_cases


def test_ties_across_the_boundary_are_kept_together():
    # four equal maxima of mass 1/4 each (+ a tail): p = 0.3 must keep all four, not stop after two
    logits = np.array([5, 5, 5, 5, -20, -20, 1], np.float32)
    keep = kept(logits, 1.0, 0, 0.3)
    assert keep[:4].all() and not keep[4:].any()
    # equal scores right below the crossing: dropped together
    logits = np.array([3.0, 1.0, 1.0, 1.0, 0.0], np.float32)
    s = logits.astype(np.float64)
    p_top = np.exp(s[0]) / np.exp(s).sum()
    keep = kept(logits, 1.0, 0, float(p_top) * 1.001)  # the maximum alone nearly reaches p
    assert keep.tolist() == [True, True, True, True, False]
    keep = kept(logits, 1.0, 0, float(p_top) * 0.5)
    assert keep.tolist() == [True, False, False, False, False]


def test_tiny_p_keeps_the_argmax_and_its_ties():
    rng = np.random.default_rng(1)
    logits = rng.standard_normal(4000).astype(np.float32)
    logits[[7, 300, 3999]] = logits.max() + 1.0
    for p in (1e-7, 1e-3, 2.0 ** -25):
        keep = kept(logits, 1.0, 0, p)
        assert np.flatnonzero(keep).tolist() == [7, 300, 3999], p


def test_top_k_one_is_greedy_for_any_p():
    rng = np.random.default_rng(2)
    for _ in range(20):
        logits = rng.standard_normal(500).astype(np.float32) * 4
        for p in (0.05, 0.5, 0.95):
            assert sampling.sample(logits, 0.9, 1, 11, 3, top_p=p) == int(np.argmax(logits))


def test_zero_mass_tokens_are_never_kept():
    # weights below 2^-32 of the maximum are mass 0, so all of Z lies above them: even p just below 1 drops
    # them (and the token of mass 1, whose own mass is below Z 2^-24), while the heavy tokens stay
    logits = np.array([0.0, -1.0, -2.0, -22.0, -23.0, -40.0], np.float32)
    q = sampling.nucleus_masses(logits)
    assert q[3] == 1 and q[4] == 0 and q[5] == 0
    for p in (float(np.nextafter(np.float32(1), np.float32(0))), 0.999999):
        keep = kept(logits, 1.0, 0, p)
        assert keep.tolist() == [True, True, True, False, False, False], p


def test_flat_vocabulary_does_not_overflow():
    V = 151936
    logits = np.full(V, 1.5, np.float32)
    u, above, z, p24, j = sampling._nucleus(logits, 0.9)
    assert z == V * 2 ** 32 and above[j] == 0
    assert kept(logits, 0.8, 0, 0.9).all()  # one run of equal scores: kept together
    logits[5] = 1.5 + 1e-3
    keep = kept(logits, 1.0, 0, 0.5)
    assert keep.sum() == V  # the maximum's mass is far below half: its followers stay with it


def test_top_p_one_is_the_old_rule_bit_for_bit():
    rng = np.random.default_rng(3)
    for V in (12, 32000):
        logits = (rng.standard_normal(V) * 3).astype(np.float32)
        for T, k in ((0.8, 0), (1.0, 40), (0.6, 5)):
            old = sampling.scores(logits, T, k, 9, 4)
            for p in (1.0, 1.5, 0.0):  # 1 is off, and only 0 < p < 1 is active
                new = sampling.scores(logits, T, k, 9, 4, top_p=p)
                assert np.array_equal(old.view(np.uint32), new.view(np.uint32))
            assert sampling.margin(logits, T, k, 9, 4) == sampling.margin(logits, T, k, 9, 4, top_p=1.0)


def test_draws_follow_the_nucleus_softmax():
    logits = np.array([2.0, 1.6, 1.5, 1.5, 0.7, 0.2, -0.5, -1.0, -3.0, -4.0, -6.0, -9.0], np.float32)
    T, p = 0.9, 0.8
    s = (logits / np.float32(T)).astype(np.float64)
    keep = kept(logits, T, 0, p)
    assert 2 < keep.sum() < len(logits)
    prob = np.where(keep, np.exp(s - s.max()), 0.0)
    prob /= prob.sum()
    n = 4000
    counts = np.bincount([sampling.sample(logits, T, 0, seed, 5, top_p=p) for seed in range(n)],
                         minlength=len(logits))
    assert counts[~keep].sum() == 0
    assert stats.chisquare(counts[keep], prob[keep] * n).pvalue > 1e-3


def test_nucleus_margin_and_size():
    logits = np.array([1.0, 1.0, 0.0], np.float32)
    assert sampling.nucleus_margin(logits, 1.0, 0, 1.0) == float("inf")
    # A of the second value is 2 q(1.0): exactly the need at p = 2 e / (2 e + 1) rounded to fp32 and 2^-24
    assert sampling.nucleus_size(logits, 1.0, 0, 0.5) == 2
    assert sampling.nucleus_size(logits, 1.0, 0, 0.95) == 3
    assert sampling.nucleus_size(logits, 1.0, 1, 0.95) == 2  # the tie at the top-k threshold
    assert sampling.nucleus_margin(logits, 1.0, 0, 0.5) > 0.1
