"""-m gpu: log-probabilities (kllm_logprobs_f32, kllm_decoder_set_logprobs / _read_logprobs / _score) against the
numpy mirror of kuiperllama_b200/sampling.py, on both engines.  Each record entry is checked against the mirror
applied to the logits obtained by stepping the same positions (kllm_decoder_logits): top-N ids exactly, lp within
the bound of DESIGN.md 5.8 for the engine's partition.

The persistent engine runs its log-probability kernel whenever they are on (set_logprobs >= 0, and every score): one
per weight format and KV cache (tests/megakernel_table.py).  The KERNEL_PAIRS tests run each of them in the fast
numerics, across a tile edge of its own attention geometry: not perturbing what the plain kernel decodes, records and
score against the mirror of the plain kernel's logits."""
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import KNOBS, engine_geometry, sequence, sms
from gpu_util import dev, ptr, sync
from megakernel_table import KV_CACHES, WEIGHT_FORMATS
from kuiperllama_b200 import KllmError, SHAPES, Decoder, check, load_library, sampling, synth_weights
from kuiperllama_b200.decoder import bf16_weights

pytestmark = pytest.mark.gpu

GRID = 132  # H100 SXM: the persistent engine's CTAs (the bound only grows with the grid)


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def make(name, numerics="exact", seed=2024):
    from kuiperllama_b200 import Decoder
    shape = SHAPES[name]
    return Decoder(shape, synth_weights(shape, "cuda", seed), numerics=numerics)


def chain(dec):
    V = dec.shape.vocab_size
    return sampling.chain_persistent(V, GRID) if dec.engine == "persistent" else sampling.chain_one_block(V)


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def check_entry(logits, k, rid, rlp, rtop, rtop_lp, top_n, what):
    """One record entry against the fp64 mirror of the raw logits of its position."""
    V = logits.shape[0]
    lp64, top, top64 = sampling.logprobs(logits, [rid], top_n)
    assert abs(rlp - lp64[0]) <= sampling.logprob_bound(lp64[0], k, V), (what, rlp, lp64[0])
    if top_n > 0:
        assert (rtop == top).all(), (what, rtop, top)
        assert np.all(np.abs(rtop_lp - top64) <= sampling.logprob_bound(top64, k, V)), what
        hit = np.flatnonzero(rtop == rid)
        if hit.size:  # the id's lp is its top-N entry, bit for bit
            assert bits(rtop_lp[hit[0]]) == bits(rlp), what


def stepped_logits(dec, tokens, start_pos):
    """Logits of each position when tokens[i] is fed at start_pos + i by kllm_decoder_step."""
    out = []
    for i, t in enumerate(tokens):
        dec.step(int(t), start_pos + i)
        out.append(dec.logits())
    return out


# ---- the per-op kernel ------------------------------------------------------------------------------------

def kernel_logprobs(lib, logits, ids, top_n):
    d = dev(logits)
    di = torch.tensor(np.asarray(ids, np.int32), device="cuda")
    lp = torch.full((max(len(ids), 1),), float("nan"), device="cuda")
    ti = torch.full((max(top_n, 1),), -7, dtype=torch.int32, device="cuda")
    tl = torch.full((max(top_n, 1),), float("nan"), device="cuda")
    check(lib.kllm_logprobs_f32(ptr(d), logits.shape[0], ptr(di), len(ids), top_n, ptr(lp), ptr(ti), ptr(tl), None),
          "kllm_logprobs_f32")
    sync()
    return lp.cpu().numpy()[:len(ids)], ti.cpu().numpy()[:top_n], tl.cpu().numpy()[:top_n]


@pytest.mark.parametrize("V", [512, 32000, 151936])
@pytest.mark.parametrize("kind", ["normal", "equal", "far", "spread"])
def test_kernel_matches_the_mirror(V, kind):
    lib = load_library()
    rng = np.random.default_rng(V)
    logits = {"normal": rng.standard_normal(V) * 4, "equal": np.full(V, 0.5),
              "far": rng.standard_normal(V), "spread": rng.uniform(-80, 80, V)}[kind].astype(np.float32)
    if kind == "far":
        logits[V // 3] = logits.max() + 60
    ids = np.concatenate([rng.integers(0, V, 40), [0, V - 1, -1, V]]).astype(np.int32)
    k = sampling.chain_one_block(V)
    for top_n in (0, 5, 20):
        lp, ti, tl = kernel_logprobs(lib, logits, ids, top_n)
        lp64, top, top64 = sampling.logprobs(logits, ids, top_n)
        ok = (ids >= 0) & (ids < V)
        assert np.isnan(lp[~ok]).all()
        assert np.all(np.abs(lp[ok] - lp64[ok]) <= sampling.logprob_bound(lp64[ok], k, V)), np.abs(lp[ok] - lp64[ok]).max()
        assert (ti == top).all(), (ti, top)
        assert np.all(np.abs(tl - top64) <= sampling.logprob_bound(top64, k, V))
        if top_n:  # one partition: the top entry and the id's lp are the same bits
            lp_top, _, _ = kernel_logprobs(lib, logits, ti.astype(np.int32), 0)
            assert (bits(lp_top) == bits(tl)).all()
    again = kernel_logprobs(lib, logits, ids, 20)
    assert all((bits(a) == bits(b)).all() for a, b in zip(again[::2], kernel_logprobs(lib, logits, ids, 20)[::2]))


def test_kernel_refusals():
    lib = load_library()
    d = dev(np.zeros(16, np.float32))
    o = torch.zeros(32, device="cuda")
    i = torch.zeros(32, dtype=torch.int32, device="cuda")
    assert lib.kllm_logprobs_f32(None, 16, ptr(i), 1, 0, ptr(o), None, None, None) == -1
    assert lib.kllm_logprobs_f32(ptr(d), 0, ptr(i), 1, 0, ptr(o), None, None, None) == -1
    assert lib.kllm_logprobs_f32(ptr(d), 16, None, 1, 0, ptr(o), None, None, None) == -1
    assert lib.kllm_logprobs_f32(ptr(d), 16, ptr(i), -1, 0, ptr(o), None, None, None) == -1
    assert lib.kllm_logprobs_f32(ptr(d), 16, ptr(i), 1, 21, ptr(o), ptr(i), ptr(o), None) == -1
    assert lib.kllm_logprobs_f32(ptr(d), 16, ptr(i), 1, -1, ptr(o), ptr(i), ptr(o), None) == -1
    assert lib.kllm_logprobs_f32(ptr(d), 16, ptr(i), 1, 3, ptr(o), None, ptr(o), None) == -1


# ---- the decoder ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["tiny", "tiny-qwen", "small", "small-int8", "small-qwen"])
@pytest.mark.parametrize("numerics", ["exact", "fast"])
def test_generate_records_match_the_mirror(engine, name, numerics):
    dec = make(name, numerics)
    assert dec.engine == engine
    n, top_n = 20, 5
    dec.set_sampling(0.9, 0, 77)
    dec.set_logprobs(top_n)
    ids = dec.generate(1, 0, n)
    rec = dec.logprobs(0, n)
    assert (rec[0] == ids).all()
    again = dec.generate(1, 0, n)  # repeated run: the same bits
    assert again == ids
    rec2 = dec.logprobs(0, n)
    assert all((np.asarray(a).view(np.uint32) == np.asarray(b).view(np.uint32)).all() for a, b in zip(rec, rec2))
    k = chain(dec)
    for pos, lg in enumerate(stepped_logits(dec, [1] + ids[:-1], 0)):
        check_entry(lg, k, rec[0][pos], rec[1][pos], rec[2][pos], rec[3][pos], top_n, (name, pos))
    # step wrote the same entries again (same engine, same logits, same draw)
    rec3 = dec.logprobs(0, n)
    assert (rec3[0] == rec[0]).all() and (bits(rec3[1]) == bits(rec[1])).all()


@pytest.mark.parametrize("name", ["small", "small-int8", "small-qwen"])
def test_engines_agree_within_the_bound(monkeypatch, name):
    recs = {}
    for eng in ("persistent", "graph"):
        monkeypatch.setenv("KLLM_ENGINE", eng)
        dec = make(name)
        dec.set_logprobs(20)
        ids = dec.generate(3, 0, 16)
        recs[eng] = (ids, dec.logprobs(0, 16))
        dec.close()
    (ia, ra), (ib, rb) = recs["persistent"], recs["graph"]
    assert ia == ib
    V = SHAPES[name].vocab_size
    k = sampling.chain_persistent(V, GRID) + sampling.chain_one_block(V)
    assert (ra[0] == rb[0]).all() and (ra[2] == rb[2]).all()
    assert np.all(np.abs(ra[1].astype(np.float64) - rb[1]) <= sampling.logprob_bound(rb[1], k, V))
    assert np.all(np.abs(ra[3].astype(np.float64) - rb[3]) <= sampling.logprob_bound(rb[3], k, V))


CONFIGS = [(0.0, 0, 1.0, 1.0), (0.8, 0, 1.0, 1.0), (0.8, 40, 1.0, 1.0), (0.8, 0, 0.9, 1.0), (0.7, 20, 0.8, 1.05),
           (0.0, 0, 1.0, 1.3)]


@pytest.mark.parametrize("name", ["small", "small-qwen"])
def test_logprobs_do_not_perturb(engine, name):
    """Ids, logits, KV cache and history bit-identical with logprobs on and off, under every sampling setting."""
    dec = make(name)
    for ci, (T, k, p, theta) in enumerate(CONFIGS):
        dec.set_sampling(T, k, 50 + ci, top_p=p)
        dec.set_repetition_penalty(theta, 0)
        out = []
        for top_n in (-1, 20, 0):
            dec.set_logprobs(top_n)
            ids = dec.generate(5, 0, 24)
            until = dec.generate_until(5, 0, 24)
            out.append((ids, until, dec.logits(), *dec.kv_cache(), dec.history()))
        for other in out[1:]:
            assert other[0] == out[0][0] and other[1] == out[0][1], (T, k, p, theta)
            for a, b in zip(other[2:], out[0][2:]):
                assert (np.asarray(a).view(np.uint32) == np.asarray(b).view(np.uint32)).all(), (T, k, p, theta)


def test_entries_only_where_the_classifier_ran(engine):
    dec = make("small")
    dec.set_logprobs(3)
    prompt = [1, 17, 300, 9, 44]
    nxt = dec.prompt(prompt)
    ids, lp, ti, tl = dec.logprobs(0, 12)
    assert (ids[:4] == -1).all() and ids[4] == nxt and (ids[5:] == -1).all()
    assert dec.step(7, 5, is_prompt=True) == -1
    assert dec.logprobs(5, 1)[0][0] == -1
    # generate_until with a stop: entries exactly where it ran
    ref = dec.generate(nxt, 5, 20)
    dec.set_logprobs(3)
    stop = ref[6]
    got = dec.generate_until(nxt, 5, 20, stop_ids=[stop])
    ids = dec.logprobs(0, 40)[0]
    assert (ids[5:5 + len(got)] == got).all() and (ids[5 + len(got):] == -1).all() and (ids[:5] == -1).all()
    # rewinding overwrites: teacher-forced generate over the same positions records the drawn ids
    teacher = [nxt] + [int(t) for t in np.random.default_rng(1).integers(0, 4096, 9)]
    drawn = dec.generate(nxt, 5, 10, teacher=teacher)
    ids = dec.logprobs(5, 10)[0]
    assert (ids == drawn).all()
    # scoring's target mode ends with the score: a generate over the same positions records the ids it drew
    tokens = [int(t) for t in np.random.default_rng(3).integers(0, 4096, 11)]
    dec.score(tokens, 5)
    assert (dec.logprobs(5, 10)[0] == tokens[1:]).all()
    drawn = dec.generate(nxt, 5, 10)
    ids = dec.logprobs(5, 10)[0]
    assert (ids == drawn).all() and (ids != tokens[1:]).any()


def test_prefill_records_the_last_position(engine):
    dec = make("small")
    dec.set_logprobs(4)
    prompt = [int(t) for t in np.random.default_rng(2).integers(0, 4096, 40)]
    nxt = dec.prefill_tf32(prompt)
    ids, lp, ti, tl = dec.logprobs(0, 41)
    assert (ids[:39] == -1).all() and ids[39] == nxt and ids[40] == -1
    check_entry(dec.logits(), chain(dec), ids[39], lp[39], ti[39], tl[39], 4, "prefill")


def test_refusals_and_clearing(engine):
    dec = make("tiny")
    dec.set_logprobs(2)
    dec.generate(1, 0, 8)
    with pytest.raises(KllmError):
        dec.set_logprobs(21)
    with pytest.raises(KllmError):
        dec.set_logprobs(-2)
    ids, _, ti, _ = dec.logprobs(0, 8)  # the setting in force (2) and the record survive a refusal
    assert (ids >= 0).all() and ti.shape == (8, 2)
    with pytest.raises(KllmError):
        dec.logprobs(60, 5)
    with pytest.raises(KllmError):
        dec.logprobs(-1, 2)
    V = dec.shape.vocab_size
    for bad, start in (([1], 0), ([1, V], 0), ([1, -1, 2], 0), ([1, 2, 3], 62), ([1, 2], -1)):
        with pytest.raises(KllmError):
            dec.score(bad, start)
    dec.set_logprobs(2)  # clears
    assert (dec.logprobs(0, 64)[0] == -1).all()


@pytest.mark.parametrize("name", ["small", "small-int8", "small-qwen"])
@pytest.mark.parametrize("numerics", ["exact", "fast"])
def test_score_matches_teacher_stepping(engine, name, numerics):
    dec = make(name, numerics)
    V = dec.shape.vocab_size
    tokens = [int(t) for t in np.random.default_rng(4).integers(0, V, 33)]
    dec.set_sampling(0.8, 40, 9)  # no effect on scoring
    dec.set_repetition_penalty(1.3, 0)
    lp = dec.score(tokens)
    assert lp.shape == (32,)
    kv_score = dec.kv_cache()
    hist = dec.history()
    assert (hist[:32] == tokens[:32]).all()
    for top_n in (-1, 6):
        dec.set_logprobs(top_n)
        again = dec.score(tokens)
        assert (bits(again) == bits(lp)).all()
    ids, rlp, ti, tl = dec.logprobs(0, 32)
    assert (ids == tokens[1:]).all() and (bits(rlp) == bits(lp)).all()
    # the same as generate(teacher) stepping + the mirror
    k = chain(dec)
    for pos, lg in enumerate(stepped_logits(dec, tokens[:32], 0)):
        check_entry(lg, k, tokens[pos + 1], lp[pos], ti[pos], tl[pos], 6, (name, pos))
    # KV cache bit-identical to kllm_decoder_prompt over the same tokens
    fresh = make(name, numerics)
    fresh.prompt(tokens[:32])
    kv_prompt = fresh.kv_cache()
    for a, b in zip(kv_score, kv_prompt):
        assert (a[:, :32].view(np.uint32) == b[:, :32].view(np.uint32)).all()
    # the sequence continues: tokens[-1] at position 32
    dec.set_sampling(0.0)
    dec.set_repetition_penalty(1.0)
    assert dec.step(tokens[32], 32) == fresh.step(tokens[32], 32)


def test_score_full_size_tinyllama(engine):
    """1 024 tokens scored on TinyLlama-1.1B's shape, against host log-softmax of the stepped logits."""
    from kuiperllama_b200 import Decoder
    shape = SHAPES["tinyllama-1.1b"]
    dec = Decoder(shape, synth_weights(shape, "cuda", 7))
    tokens = [int(t) for t in np.random.default_rng(8).integers(0, shape.vocab_size, 1025)]
    lp = dec.score(tokens)
    k = chain(dec)
    for pos in range(0, 1024, 1):
        dec.step(tokens[pos], pos)
        if pos % 8 == 0 or pos == 1023:
            lg = dec.logits().astype(np.float64)
            m = lg.max()
            want = lg[tokens[pos + 1]] - m - np.log(np.exp(lg - m).sum())
            assert abs(lp[pos] - want) <= sampling.logprob_bound(want, k, shape.vocab_size), (pos, lp[pos], want)


# ---- every log-probability kernel of the persistent engine ----------------------------------------------------------
# (weight format, KV cache): every pair the persistent engine has kernels for, at small-int8's dimensions (head_size 64,
# two query heads per KV head), the fp32 and bf16 weights built at the same dimensions without int8 groups.  Flash
# tiles (engine_geometry): 64 / 256 / 256 timesteps for fp32 weights over the fp32 / bf16 / fp8 caches, 96 / 192 / 256
# for int8 and for bf16 weights.
KERNEL_PAIRS = [(f, kv) for f in WEIGHT_FORMATS for kv in KV_CACHES]
PAIR_SHAPE = replace(SHAPES["small-int8"], seq_len=320)
PENALISED = (0.8, 40, 0.9, 1.3)  # temperature, top-k, top-p, repetition penalty


def pair_id(p):
    return f"{p[0]}w-{p[1]}kv"


@pytest.fixture(scope="module")
def pair_weights():
    fp32 = synth_weights(replace(PAIR_SHAPE, group_size=0), "cuda", 2024)
    return {"fp32": fp32, "int8": synth_weights(PAIR_SHAPE, "cuda", 2024), "bf16": bf16_weights(fp32)}


def make_pair(monkeypatch, pair_weights, weight_format, kv_cache):
    """The persistent engine in the fast numerics with `weight_format` weights over a `kv_cache` cache (fp8 at a
    scale of 0.02); its attention geometry must be engine_geometry's."""
    for name in KNOBS:
        monkeypatch.delenv(name, raising=False)
    monkeypatch.setenv("KLLM_ENGINE", "persistent")
    shape = PAIR_SHAPE if weight_format == "int8" else replace(PAIR_SHAPE, group_size=0)
    sc = np.full((2, shape.layer_num, shape.kv_head_num), 0.02, np.float32) if kv_cache == "fp8" else None
    dec = Decoder(shape, pair_weights[weight_format], numerics="fast", kv_cache=kv_cache, kv_scales=sc,
                  weight_format="bf16" if weight_format == "bf16" else "fp32")
    assert dec.engine == "persistent"
    assert dec.attention_geometry == engine_geometry(shape, "fast", {}, sms(), kv_cache, weight_format), \
        (weight_format, kv_cache, dec.attention_geometry)
    return dec


@pytest.mark.parametrize("weight_format,kv_cache", KERNEL_PAIRS, ids=[pair_id(p) for p in KERNEL_PAIRS])
def test_kernel_pair_logprobs_do_not_perturb(monkeypatch, pair_weights, weight_format, kv_cache):
    """Teacher-forced generate over the first tile and three positions past it, greedy and sampled-and-penalised (the
    penalised classifier partials are the log-probability kernel's own branch): ids, logits, cache rows and history
    bit-identical with log-probabilities off (the plain kernel), on without alternatives and on with 20."""
    dec = make_pair(monkeypatch, pair_weights, weight_format, kv_cache)
    T = dec.attention_geometry[0]
    V = dec.shape.vocab_size
    toks = sequence(V, T + 3, 11)
    for temperature, top_k, top_p, theta in ((0.0, 0, 1.0, 1.0), PENALISED):
        dec.set_sampling(temperature, top_k, 50, top_p=top_p)
        dec.set_repetition_penalty(theta, 0)
        out = []
        for top_n in (-1, 0, 20):
            dec.set_logprobs(top_n)
            ids = dec.generate(0, 0, len(toks), teacher=toks)
            out.append((ids, dec.logits(), *dec.kv_cache(), dec.history()))
        for top_n, other in zip((0, 20), out[1:]):
            what = (weight_format, kv_cache, temperature, top_n)
            assert other[0] == out[0][0], what
            for a, b in zip(other[1:], out[0][1:]):
                assert (np.asarray(a).view(np.uint32) == np.asarray(b).view(np.uint32)).all(), what
    dec.close()


@pytest.mark.parametrize("weight_format,kv_cache", KERNEL_PAIRS, ids=[pair_id(p) for p in KERNEL_PAIRS])
def test_kernel_pair_records_match_the_mirror(monkeypatch, pair_weights, weight_format, kv_cache):
    """Sampled generate across the first tile edge with 5 alternatives recorded; each entry against the mirror of the
    logits the plain kernel gives when it steps the same ids at the same positions."""
    dec = make_pair(monkeypatch, pair_weights, weight_format, kv_cache)
    T = dec.attention_geometry[0]
    V = dec.shape.vocab_size
    start, n, top_n = T - 8, 16, 5
    dec.set_logprobs(top_n)
    dec.set_sampling(0.9, 0, 77)
    nxt = dec.prompt(sequence(V, start, 12))
    ids = dec.generate(nxt, start, n)
    rec = dec.logprobs(start, n)
    assert (rec[0] == ids).all()
    dec.set_logprobs(-1)
    k = sampling.chain_persistent(V, GRID)
    for i, lg in enumerate(stepped_logits(dec, [nxt] + ids[:-1], start)):
        check_entry(lg, k, rec[0][i], rec[1][i], rec[2][i], rec[3][i], top_n, (weight_format, kv_cache, start + i))
    dec.close()


@pytest.mark.parametrize("weight_format,kv_cache", KERNEL_PAIRS, ids=[pair_id(p) for p in KERNEL_PAIRS])
def test_kernel_pair_score_matches_teacher_stepping(monkeypatch, pair_weights, weight_format, kv_cache):
    """score over the first tile and past its edge, sampled and penalised settings in force (no effect on scoring):
    each value and its alternatives against the mirror of the plain kernel's stepped logits, and the cache rows bit for
    bit those prompt writes over the same tokens."""
    dec = make_pair(monkeypatch, pair_weights, weight_format, kv_cache)
    T = dec.attention_geometry[0]
    V = dec.shape.vocab_size
    tokens = sequence(V, T + 4, 4)
    n = len(tokens) - 1
    dec.set_sampling(0.8, 40, 9)
    dec.set_repetition_penalty(1.3, 0)
    dec.set_logprobs(6)
    lp = dec.score(tokens)
    assert lp.shape == (n,)
    ids, rlp, ti, tl = dec.logprobs(0, n)
    assert (ids == tokens[1:]).all() and (bits(rlp) == bits(lp)).all()
    kv_score = dec.kv_cache()
    dec.set_logprobs(-1)
    dec.set_sampling(0.0)
    dec.set_repetition_penalty(1.0)
    k = sampling.chain_persistent(V, GRID)
    for pos, lg in enumerate(stepped_logits(dec, tokens[:n], 0)):
        check_entry(lg, k, tokens[pos + 1], lp[pos], ti[pos], tl[pos], 6, (weight_format, kv_cache, pos))
    fresh = make_pair(monkeypatch, pair_weights, weight_format, kv_cache)
    fresh.prompt(tokens[:n])
    for a, b in zip(kv_score, fresh.kv_cache()):
        assert (a[:, :n].view(np.uint32) == b[:, :n].view(np.uint32)).all(), (weight_format, kv_cache)
    dec.close()
    fresh.close()
