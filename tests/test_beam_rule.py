"""CPU: the beam-search rule of kuiperllama_b200/beam.py (kllm_batch_beam_search's) bit for bit against the installed
transformers' GenerationMixin._beam_search, over seeded fp32 log-probability tables that replace a tiny model's, and
its edge cases by construction."""
import zlib
from unittest import mock

import numpy as np
import pytest

from kuiperllama_b200 import beam

V = 48  # >= K = max(2, 1 + n_eos) * B for every case below


def table(prefix, seed, eos=(), eos_depths=()):
    """The log-probabilities after the generated ids `prefix`: a seeded fp32 row in (-12, 0), with the eos ids made
    likely at the depths in eos_depths"""
    key = zlib.crc32(np.asarray([seed] + list(prefix), np.int64).tobytes())
    rng = np.random.default_rng(key)
    row = (-rng.uniform(0.05, 12.0, V)).astype(np.float32)
    if len(prefix) in eos_depths:
        for j, e in enumerate(eos):
            row[e] = np.float32(-0.01 * (j + 1) - rng.uniform(0, 0.02))
    return row


def order(row):
    """The logprob rule's top-N order of a row: value descending, lowest id on ties"""
    return sorted(range(len(row)), key=lambda i: (-row[i], i))


def mirror(n_beams, max_new, eos, alpha, early, n_return, seed, eos_depths, start_pos=0):
    def candidates(beams):
        out = []
        for b in beams:
            row = table(b.ids, seed, eos, eos_depths)
            ids = order(row)[:n_beams + len(eos)]
            out.append((ids, row[ids]))
        return out
    return beam.beam_search(candidates, n_beams, max_new, eos, alpha, early, n_return, start_pos)


def hf_generate(n_beams, max_new, eos, alpha, early, n_return, seed, eos_depths):
    transformers = pytest.importorskip("transformers")
    torch = pytest.importorskip("torch")
    torch.manual_seed(0)
    cfg = transformers.LlamaConfig(vocab_size=V, hidden_size=16, intermediate_size=32, num_hidden_layers=1,
                                   num_attention_heads=2, num_key_value_heads=1, max_position_embeddings=64,
                                   bos_token_id=None, eos_token_id=None, pad_token_id=None)
    model = transformers.LlamaForCausalLM(cfg).eval()
    prompt_len = 3

    class Table(transformers.LogitsProcessor):
        def __call__(self, input_ids, scores):
            rows = [table(tuple(int(x) for x in seq[prompt_len:]), seed, eos, eos_depths) for seq in input_ids]
            return torch.tensor(np.stack(rows))

    gc = transformers.GenerationConfig(num_beams=n_beams, do_sample=False, max_new_tokens=max_new,
                                       eos_token_id=list(eos) if eos else None, pad_token_id=0,
                                       length_penalty=alpha, early_stopping=early, num_return_sequences=n_return,
                                       return_dict_in_generate=True, output_scores=True)
    # transformers runs one beam as greedy search: its _beam_search is selected explicitly for B = 1
    mode = transformers.generation.configuration_utils.GenerationMode.BEAM_SEARCH
    with torch.no_grad(), mock.patch.object(transformers.GenerationConfig, "get_generation_mode",
                                            lambda *args, **kwargs: mode):
        out = model.generate(torch.tensor([[5, 6, 7]]), generation_config=gc,
                             logits_processor=transformers.LogitsProcessorList([Table()]))
    seqs = out.sequences[:, prompt_len:].numpy()
    lens = (out.beam_indices >= 0).sum(dim=1).numpy()
    return [(list(seqs[i, :lens[i]]), np.float32(out.sequences_scores[i].item())) for i in range(n_return)]


def bits(x):
    return np.float32(x).view(np.uint32)


def check_against_hf(B, n_eos, alpha, early, max_new, seed):
    eos = [40 + j for j in range(n_eos)]
    depths = {1, 3} if seed % 2 else {0, 2, 4}
    hf = hf_generate(B, max_new, eos, alpha, early, B, seed, depths)
    ours, _ = mirror(B, max_new, eos, alpha, early, B, seed, depths)
    assert len(ours) == B
    for (ids, score), h in zip(hf, ours):
        assert h["ids"] == [int(i) for i in ids]
        assert bits(h["score"]) == bits(score), (h["score"], score)


@pytest.mark.parametrize("B", range(1, 9))
@pytest.mark.parametrize("n_eos", range(4))
@pytest.mark.parametrize("early", [False, True, "never"])
def test_rule_is_transformers_bit_for_bit(B, n_eos, early):
    """Every returned sequence and sequences_score, all B of them (so every n_return's prefix), across the length
    penalties; eos ids made likely at some depths so that hypotheses finish early"""
    for k, alpha in enumerate([-0.5, 0.0, 1.0, 2.0]):
        check_against_hf(B, n_eos, alpha, early, 6, seed=100 * B + 10 * n_eos + k)


@pytest.mark.parametrize("B", [1, 2, 5, 8])
@pytest.mark.parametrize("early", [False, True, "never"])
def test_one_new_token(B, early):
    for alpha in [-0.5, 1.0]:
        check_against_hf(B, 1, alpha, early, 1, seed=7 + B)


@pytest.mark.parametrize("n_return", [1, 2, 4])
def test_n_return_is_the_best_prefix(n_return):
    """num_return_sequences < num_beams: transformers' first n_return, and the mirror's"""
    eos, depths = [41, 42], {1, 3}
    hf = hf_generate(4, 6, eos, 1.0, False, n_return, 3, depths)
    ours, _ = mirror(4, 6, eos, 1.0, False, n_return, 3, depths)
    assert [h["ids"] for h in ours] == [[int(i) for i in ids] for ids, _ in hf]
    assert [bits(h["score"]) for h in ours] == [bits(s) for _, s in hf]


def test_torch_divides_in_float32():
    """h = fp32(s / fp32(t ** alpha)): torch rounds the Python float to float32 and divides in float32"""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(5)
    s = (rng.standard_normal(100000) * 40).astype(np.float32)
    for t in [1, 2, 3, 7, 64, 511]:
        for alpha in [-0.5, 0.0, 0.7, 1.0, 2.0]:
            hf = (torch.from_numpy(s) / (t ** alpha)).numpy()
            assert (hf.view(np.uint32) == (s / beam.length_divisor(t, alpha)).view(np.uint32)).all()


def fixed(rows):
    """candidates() over fixed rows per depth: rows[len(ids)] is (ids, lp) for every beam at that depth"""
    return lambda beams: [rows[len(b.ids)] for b in beams]


def test_eos_beyond_rank_b_is_not_offered():
    """An eos candidate at rank >= B is not a hypothesis, and no next beam"""
    B = 2
    rows = {0: ([3, 4, 9], np.float32([-0.1, -0.2, -0.3])),
            1: ([5, 6, 9], np.float32([-1.0, -1.1, -1.2])),
            2: ([7, 8, 9], np.float32([-1.0, -2.0, -3.0]))}
    hyps, _ = beam.beam_search(fixed(rows), B, 3, eos_ids=[9], length_penalty=0.0, n_return=2)
    assert all(9 not in h["ids"] for h in hyps)
    assert [h["ids"] for h in hyps] == [[3, 5, 7], [3, 6, 7]]


def test_all_top_b_eos():
    """Every one of the first B ranks an eos id: all become hypotheses, and the next beams are the best non-eos ids"""
    B = 2
    rows = {0: ([8, 9, 3, 4], np.float32([-0.1, -0.2, -0.5, -0.6])),
            1: ([8, 9, 5, 6], np.float32([-3.0, -3.1, -3.2, -3.3])),
            2: ([5, 6, 8, 9], np.float32([-0.1, -0.2, -0.3, -0.4]))}
    hyps, stats = beam.beam_search(fixed(rows), B, 3, eos_ids=[8, 9], length_penalty=1.0, n_return=2)
    assert [h["ids"] for h in hyps] == [[8], [9]]
    assert bits(hyps[0]["score"]) == bits(np.float32(-0.1))
    # after pass 0 both slots are full and -0.5 / 1 < -0.2: the heuristic is satisfied and the search stops
    assert stats == {"passes": 1, "forks": 1, "fork_rows": 1}


def test_exact_ties_follow_the_stated_order():
    """Equal s: beam index ascending, then the beam's own order; equal h: the held slot first"""
    B = 3
    rows = {0: ([1, 2, 3], np.float32([-1.0, -2.0, -3.0])),
            1: ([4, 5, 6], np.float32([-1.0, -1.0, -1.0]))}
    hyps, stats = beam.beam_search(fixed(rows), B, 2, length_penalty=0.0, n_return=3)
    # pass 1: beams (1,), (2,), (3,) at -1, -2, -3; each offers 4, 5, 6 at S - 1: the top 3 are all of beam 0, in
    # its own order
    assert [h["ids"] for h in hyps] == [[1, 4], [1, 5], [1, 6]]
    assert stats["passes"] == 2 and stats["forks"] == 2
    # a held slot ahead of an equal offer
    rows = {0: ([7, 1, 2], np.float32([-1.0, -1.0, -5.0])),
            1: ([7, 3, 4], np.float32([0.0, -1.0, -1.0]))}
    hyps, _ = beam.beam_search(fixed(rows), 2, 2, eos_ids=[7], length_penalty=0.0, early_stopping="never",
                               n_return=2)
    assert hyps[0]["ids"] == [7]
    assert bits(hyps[0]["score"]) == bits(hyps[1]["score"])


def test_fork_stats():
    """Forks per pass: B - 1 prompt copies after pass 0, then B - distinct parents of t - 1 generated rows"""
    B = 3
    rows = {d: ([10 + d, 20 + d, 30 + d], np.float32([-1.0, -1.5, -9.0])) for d in range(4)}
    hyps, stats = beam.beam_search(fixed(rows), B, 4, length_penalty=0.0, start_pos=5)
    # passes 1 .. 2 keep the best two children of beam 0 and one of beam 1: 2 distinct parents, 1 fork each
    assert stats["passes"] == 4
    assert stats["forks"] == 2 + 1 + 1
    assert stats["fork_rows"] == 2 * 6 + 1 * 1 + 1 * 2
