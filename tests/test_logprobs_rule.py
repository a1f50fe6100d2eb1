"""The logprob rule (csrc/sampling.cuh, DESIGN.md 5.8) on the CPU: the numpy mirror against torch's fp64
log_softmax / topk, and the fp32 emulation of L1-L3 over a partition within the stated bound of fp64, for the
partitions the engines use and adversarial vectors."""
import numpy as np
import pytest
import torch

from kuiperllama_b200 import sampling


def fp64_reference(logits, ids, n):
    t = torch.tensor(np.asarray(logits, np.float32), dtype=torch.float64)
    lsm = torch.log_softmax(t, 0).numpy()
    return lsm[np.asarray(ids, np.int64)], lsm


def random_parts(V, n_parts, rng):
    cuts = np.sort(rng.choice(np.arange(1, V), size=min(n_parts, V) - 1, replace=False))
    edges = np.concatenate([[0], cuts, [V]])
    return list(zip(edges[:-1].tolist(), edges[1:].tolist()))


def even_parts(V, n_parts):
    return [(c * V // n_parts, (c + 1) * V // n_parts) for c in range(n_parts)]


def check_within_bound(logits, parts, top_n=20, ids=None):
    V = logits.shape[0]
    k = sampling.chain_of_parts(parts)
    ids = np.arange(0, V, max(1, V // 97)) if ids is None else ids
    lp, top, lp_top = sampling.logprobs(logits, ids, top_n, parts)
    ref_ids, lsm = fp64_reference(logits, ids, V)
    assert np.all(np.abs(lp - ref_ids) <= sampling.logprob_bound(ref_ids, k, V)), np.max(np.abs(lp - ref_ids))
    ref_top = sampling.top_n(logits, top_n)
    assert (top == ref_top).all()
    valid = ref_top >= 0
    assert np.all(np.abs(lp_top[valid] - lsm[ref_top[valid]]) <= sampling.logprob_bound(lsm[ref_top[valid]], k, V))
    return lp, top, lp_top


def test_mirror_fp64_equals_torch():
    rng = np.random.default_rng(0)
    logits = (rng.standard_normal(4096) * 3).astype(np.float32)
    ids = rng.integers(0, 4096, 50)
    lp, top, lp_top = sampling.logprobs(logits, ids, 20)
    ref, lsm = fp64_reference(logits, ids, 4096)
    np.testing.assert_allclose(lp, ref, rtol=0, atol=1e-12)
    vals, idx = torch.topk(torch.tensor(logits, dtype=torch.float64), 20)
    assert (top == idx.numpy()).all()  # distinct values: topk's order is the rule's
    np.testing.assert_allclose(lp_top, lsm[top], rtol=0, atol=1e-12)


def test_tie_rule_lowest_index_first():
    logits = np.zeros(64, np.float32)
    logits[[5, 9, 40]] = 2.0
    logits[[3, 7]] = 1.0
    top = sampling.top_n(logits, 8)
    assert top.tolist() == [5, 9, 40, 3, 7, 0, 1, 2]
    assert sampling.top_n(logits[:4], 6).tolist() == [3, 0, 1, 2, -1, -1]


@pytest.mark.parametrize("V", [512, 32000, 151936])
@pytest.mark.parametrize("n_parts", [1, 32, 132, 1024])
def test_fp32_partitions_within_bound(V, n_parts):
    rng = np.random.default_rng(V + n_parts)
    logits = (rng.standard_normal(V) * 4).astype(np.float32)
    check_within_bound(logits, random_parts(V, n_parts, rng))
    check_within_bound(logits, even_parts(V, n_parts))


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_all_equal(V):
    logits = np.full(V, 1.25, np.float32)
    for parts in (even_parts(V, 132), sampling.warp_parts(V)):
        lp, top, lp_top = check_within_bound(logits, parts)
        assert top.tolist() == list(range(20))
        assert np.all(np.abs(lp_top + np.log(V)) <= sampling.logprob_bound(np.log(V), sampling.chain_of_parts(parts), V))


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_one_logit_far_above(V):
    rng = np.random.default_rng(7)
    logits = rng.standard_normal(V).astype(np.float32)
    logits[V // 3] = 60.0 + logits.max()
    lp, top, lp_top = check_within_bound(logits, even_parts(V, 132), ids=[V // 3, 0, V - 1])
    assert top[0] == V // 3 and abs(lp_top[0]) < 1e-6


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_spread_of_80(V):
    rng = np.random.default_rng(11)
    logits = rng.uniform(-80, 80, V).astype(np.float32)
    for n_parts in (1, 132, 1024):
        check_within_bound(logits, random_parts(V, n_parts, rng))


def test_top_n_larger_than_a_part():
    # ~4 rows per part (the tiny test models on 132 CTAs): N = 20 spans several parts
    V = 512
    rng = np.random.default_rng(3)
    logits = (rng.standard_normal(V) * 2).astype(np.float32)
    logits[100:140] = 20.0  # ties across many parts
    lp, top, lp_top = check_within_bound(logits, even_parts(V, 132))
    assert top.tolist() == list(range(100, 120))


@pytest.mark.parametrize("V", [512, 32000, 151936])
def test_engine_chains_within_the_target(V):
    """The engines' chains keep the derived bound near 1e-5 + 1e-6 |lp| (the target): at most 1.6e-5 at lp = 0."""
    for k in (sampling.chain_persistent(V, 132), sampling.chain_one_block(V)):
        assert sampling.logprob_bound(0.0, k, V) <= 1.6e-5
        assert sampling.logprob_bound(-50.0, k, V) <= 1e-5 + 1e-6 * 50


def test_same_partition_same_bits():
    rng = np.random.default_rng(5)
    logits = (rng.standard_normal(32000) * 3).astype(np.float32)
    parts = even_parts(32000, 132)
    a = sampling.logprobs(logits, [1, 2, 3], 5, parts)
    b = sampling.logprobs(logits, [1, 2, 3], 5, parts)
    assert all((x.view(np.uint64) == y.view(np.uint64)).all() for x, y in zip(a, b))
