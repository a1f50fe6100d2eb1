"""-m gpu: a batch of decoders over one model (kllm_batch) against twin decoders over the same weights that run their
own entries, bit for bit: ids, logits, history, log-probability record (with the persistent engine's last-bits
exception on the log-probabilities) and the KV rows up to each member's frontier; and kllm_decoder_copy_prefix on
every engine and cache."""
import ctypes
from dataclasses import replace

import numpy as np
import pytest

from decode_model_util import GEOMETRIES
from gpu_util import assert_bit_equal
from kuiperllama_b200 import MAX_BATCH, SHAPES, Batch, Decoder, KllmError, ModelShape, synth_weights
from kuiperllama_b200.decoder import bf16_weights

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -2

# shapes only the graph engine takes (as in test_speculative_gpu.py): head_size 256, int8 scale rows of 36 bytes,
# seq_len % 4 != 0
GRAPH_ONLY = {
    "hs256": ModelShape("hs256", 512, 1376, 2, 2, 1, 1024, 544),
    "int8-g32-hs48": ModelShape("int8-g32-hs48", 288, 768, 2, 6, 2, 1024, 544, group_size=32),
    "seq1001": replace(SHAPES["small"], name="small-seq1001", seq_len=1001),
}


@pytest.fixture(params=["persistent", "graph"])
def engine(request, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", request.param)
    return request.param


def decoders(shape, engine, n, weight_format="fp32", seed=2024, top_n=5):
    """n members and n twins over one weight set, each with logprobs top_n."""
    w = synth_weights(shape, "cuda", seed)
    if weight_format == "bf16":
        w = bf16_weights(w)
    try:
        ds = [Decoder(shape, w, weight_format=weight_format) for _ in range(2 * n)]
    except KllmError:
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    if ds[0].engine != engine:
        pytest.skip(f"{shape.name}: the {engine} engine does not take this shape")
    for d in ds:
        d.set_logprobs(top_n)
    return ds[:n], ds[n:]


def assert_same_state(a, b, upto, what, lp_exception=True):
    """a ran batch entries, b its own: logits, history and record over the whole sequence, KV rows below upto."""
    assert_bit_equal(a.logits(), b.logits(), f"{what}: logits")
    assert np.array_equal(a.history(), b.history()), f"{what}: history"
    n = a.shape.seq_len
    for x, y, name in zip(a.logprobs(0, n), b.logprobs(0, n), ("ids", "lp", "top_ids", "top_lp")):
        if lp_exception and a.engine == "persistent" and name in ("lp", "top_lp"):
            # the megakernel sums the log-softmax normaliser from per-CTA partials; the chain's draw sums it in
            # argmax_advance_kernel's order, so the log-probabilities may differ in the last bits (DESIGN.md 5.14)
            np.testing.assert_allclose(x, y, rtol=2e-6, atol=0, err_msg=f"{what}: record {name}")
        else:
            assert_bit_equal(x, y, f"{what}: record {name}")
    for x, y in zip(a.kv_cache(), b.kv_cache()):
        assert_bit_equal(x[:, :upto], y[:, :upto], f"{what}: kv rows")


def batch_vs_twins(members, twins, firsts, positions, k, what=""):
    """One Batch.generate of k steps against each twin's own generate; returns the ids."""
    batch = Batch(members)
    try:
        ids = batch.generate(firsts, positions, k)
    finally:
        batch.close()
    for b, (m, t) in enumerate(zip(members, twins)):
        assert t.generate(firsts[b], positions[b], k) == ids[b], f"{what} member {b}: ids"
        assert_same_state(m, t, positions[b] + k, f"{what} member {b}")
    return ids


def prefill(members, twins, lengths, vocab):
    """Member b and its twin fed a prompt of lengths[b] ids; returns the ids each continues with."""
    firsts = []
    for b, (m, t) in enumerate(zip(members, twins)):
        L = lengths[b]
        if L == 0:
            firsts.append((7 * b + 1) % vocab)
            continue
        prompt = [(11 * b + 3 * i + 1) % vocab for i in range(L)]
        nxt = m.prompt(prompt, 0)
        assert t.prompt(prompt, 0) == nxt
        firsts.append(nxt)
    return firsts


@pytest.mark.parametrize("key", list(GEOMETRIES))
def test_batch_generate_on_every_geometry(kllm_lib, engine, key):
    """B = 1, 2, 3 and 8 in turn over the same members, whose prompts differ in length."""
    shape = GEOMETRIES[key]
    members, twins = decoders(shape, engine, MAX_BATCH)
    lengths = [min(3 + 7 * b, shape.seq_len // 4) for b in range(MAX_BATCH)]
    firsts = prefill(members, twins, lengths, shape.vocab_size)
    pos = list(lengths)
    big = shape.layer_num * shape.dim > 2048 * 4
    k = 3 if big else 6
    for B in (1, 2, 3, 8):
        ids = batch_vs_twins(members[:B], twins[:B], firsts[:B], pos[:B], k, f"B={B}")
        for b in range(B):
            firsts[b], pos[b] = ids[b][-1], pos[b] + k


SETTINGS = [
    lambda d: None,  # greedy
    lambda d: d.set_sampling(0.8, 40, 1234),
    lambda d: d.set_sampling(0.9, 0, 77, top_p=0.85),
    lambda d: d.set_repetition_penalty(1.3, 16),
    lambda d: d.set_frequency_presence(0.5, 0.4, 20),
    lambda d: d.set_logit_bias({5: 3.0, 17: -100.0, 42: 2.5}),
    lambda d: d.set_logprobs(5),
    lambda d: (d.set_sampling(1.1, 0, 2**40 + 3, top_p=0.9), d.set_repetition_penalty(0.8, 0),
               d.set_frequency_presence(-0.3, 0.2, 0), d.set_logit_bias({9: 4.0})),
]


def test_each_member_draws_under_its_own_settings(kllm_lib, engine):
    shape = SHAPES["small"]
    members, twins = decoders(shape, engine, MAX_BATCH, top_n=-1)
    for b, (m, t) in enumerate(zip(members, twins)):
        SETTINGS[b](m), SETTINGS[b](t)
    firsts = prefill(members, twins, [20 + b for b in range(MAX_BATCH)], shape.vocab_size)
    pos = [20 + b for b in range(MAX_BATCH)]
    ids = batch_vs_twins(members, twins, firsts, pos, 24, "settings")
    assert len({tuple(r) for r in ids}) > 1


@pytest.mark.parametrize("key,weight_format,full", [
    ("small-int8", "fp32", False), ("int8-g32", "fp32", False), ("small", "bf16", False),
    ("tinyllama-1.1b", "bf16", True), ("small-qwen", "fp32", False), ("w2-groups", "fp32", False),
])
def test_weight_formats_and_shapes(kllm_lib, engine, key, weight_format, full):
    extra = {
        "int8-g32": ModelShape("int8-g32", 256, 768, 2, 4, 2, 1024, 160, group_size=32),
        # a small dim beside hidden_dim 11008: W2's rows split into groups at B >= 5
        "w2-groups": ModelShape("w2-groups", 256, 11008, 2, 4, 2, 1024, 192),
    }
    shape = extra.get(key) or SHAPES[key]
    if not full:
        shape = replace(shape, seq_len=min(shape.seq_len, 256))
    members, twins = decoders(shape, engine, MAX_BATCH, weight_format)
    lengths = [2 + 5 * b for b in range(MAX_BATCH)]
    firsts = prefill(members, twins, lengths, shape.vocab_size)
    for B in (5, 8):
        ids = batch_vs_twins(members[:B], twins[:B], firsts[:B], lengths[:B], 4, f"{key} B={B}")
        for b in range(B):
            firsts[b], lengths[b] = ids[b][-1], lengths[b] + 4


@pytest.mark.parametrize("key", list(GRAPH_ONLY))
def test_graph_only_shapes(kllm_lib, monkeypatch, key):
    monkeypatch.setenv("KLLM_ENGINE", "graph")
    shape = GRAPH_ONLY[key]
    members, twins = decoders(shape, "graph", 4)
    S = shape.seq_len
    lengths = [0, 9, S - 300, S - 6]  # the cache's last rows, and members far apart
    firsts = prefill(members, twins, lengths, shape.vocab_size)
    batch_vs_twins(members, twins, firsts, lengths, 6, key)


def test_edges_of_the_sequence(kllm_lib, engine):
    """A member at position 0, one whose last step is at seq_len - 1, members more than 256 positions apart, and a
    member rewound over a stale cache."""
    shape = replace(SHAPES["small"], seq_len=640)
    S = shape.seq_len
    members, twins = decoders(shape, engine, 4)
    # member 3 ran further once, then is rewound: its cache holds rows past the position it restarts from
    for d in (members[3], twins[3]):
        d.generate(5, 0, 400)
    lengths = [0, 1, S - 5, 300]
    firsts = prefill(members, twins, lengths, shape.vocab_size)
    batch_vs_twins(members, twins, firsts, lengths, 5, "edges")


def test_batch_interleaved_with_own_entries(kllm_lib, engine):
    """Batch, own generate, batch again; a member in two batches in turn; batches destroyed and re-created."""
    shape = SHAPES["small"]
    members, twins = decoders(shape, engine, 4)
    lengths = [4, 9, 15, 30]
    firsts = prefill(members, twins, lengths, shape.vocab_size)
    pos = list(lengths)
    ab, cd = Batch(members[:2]), Batch([members[1], members[2], members[3]])
    ids = ab.generate(firsts[:2], pos[:2], 5)
    for b in range(2):
        assert twins[b].generate(firsts[b], pos[b], 5) == ids[b]
        firsts[b], pos[b] = ids[b][-1], pos[b] + 5
    # member 1 on its own
    own = members[1].generate(firsts[1], pos[1], 3)
    assert twins[1].generate(firsts[1], pos[1], 3) == own
    firsts[1], pos[1] = own[-1], pos[1] + 3
    # member 1 in the other batch
    ids = cd.generate(firsts[1:], pos[1:], 4)
    for b in range(1, 4):
        assert twins[b].generate(firsts[b], pos[b], 4) == ids[b - 1]
        firsts[b], pos[b] = ids[b - 1][-1], pos[b] + 4
    ab.close()
    ids = cd.generate(firsts[1:], pos[1:], 2)
    for b in range(1, 4):
        assert twins[b].generate(firsts[b], pos[b], 2) == ids[b - 1]
        firsts[b], pos[b] = ids[b - 1][-1], pos[b] + 2
    cd.close()
    ab = Batch(members[:2])  # re-created
    ids = ab.generate(firsts[:2], pos[:2], 3)
    ab.close()
    for b in range(2):
        assert twins[b].generate(firsts[b], pos[b], 3) == ids[b]
        pos[b] += 3
    for b in range(4):
        assert_same_state(members[b], twins[b], pos[b], f"interleaved member {b}")


def test_batch_step_equals_decoder_step(kllm_lib, engine):
    shape = SHAPES["small"]
    members, twins = decoders(shape, engine, 3)
    members[1].set_sampling(0.7, 20, 99), twins[1].set_sampling(0.7, 20, 99)
    pos = [0, 17, 60]
    tokens = [3, 4, 5]
    batch = Batch(members)
    for _ in range(4):
        nxt = batch.step(tokens, pos)
        for b in range(3):
            assert twins[b].step(tokens[b], pos[b]) == nxt[b]
        tokens, pos = nxt, [p + 1 for p in pos]
    batch.close()
    for b in range(3):
        assert_same_state(members[b], twins[b], pos[b], f"step member {b}")


def snapshot(d):
    n = d.shape.seq_len
    return d.logits(), d.history(), d.logprobs(0, n), d.kv_cache()


def assert_unchanged(d, snap, what):
    logits, hist, rec, kv = snapshot(d)
    assert_bit_equal(logits, snap[0], f"{what}: logits")
    assert np.array_equal(hist, snap[1]), f"{what}: history"
    for x, y in zip(rec, snap[2]):
        assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                              y.view(np.uint32) if y.dtype == np.float32 else y), f"{what}: record"
    for x, y in zip(kv, snap[3]):
        assert_bit_equal(x, y, f"{what}: cache")


def create_rc(lib, ds, n=None):
    arr = (ctypes.c_void_p * max(len(ds), 1))(*[d.handle.value if d is not None else None for d in ds])
    out = ctypes.c_void_p()
    rc = lib.kllm_batch_create(arr, len(ds) if n is None else n, None, ctypes.byref(out))
    if rc == 0:
        lib.kllm_batch_destroy(out)
    return rc


def test_refusals_leave_every_member_unchanged(kllm_lib, engine, monkeypatch):
    shape = SHAPES["small"]
    S, V = shape.seq_len, shape.vocab_size
    w = synth_weights(shape, "cuda", 2024)
    a, b = Decoder(shape, w), Decoder(shape, w)
    if a.engine != engine:
        pytest.skip("engine")
    for d in (a, b):
        d.set_logprobs(2)
        d.generate(3, 0, 20)
    snaps = [snapshot(a), snapshot(b)]
    lib = a.lib
    nine = [Decoder(shape, w) for _ in range(7)] + [a, b]
    assert create_rc(lib, nine) == E_INVALID
    assert create_rc(lib, [a], n=0) == E_INVALID
    assert create_rc(lib, [a, None]) == E_INVALID
    assert create_rc(lib, [a, a]) == E_INVALID
    out = ctypes.c_void_p()
    assert lib.kllm_batch_create(None, 1, None, ctypes.byref(out)) == E_INVALID
    arr = (ctypes.c_void_p * 1)(a.handle.value)
    assert lib.kllm_batch_create(arr, 1, None, None) == E_INVALID
    # another weight set
    other = Decoder(shape, synth_weights(shape, "cuda", 2025))
    assert create_rc(lib, [a, other]) == E_UNSUPPORTED
    # a graph member beside a persistent one
    monkeypatch.setenv("KLLM_ENGINE", "graph" if engine == "persistent" else "persistent")
    flip = Decoder(shape, w)
    assert flip.engine != engine
    assert create_rc(lib, [a, flip]) == E_UNSUPPORTED
    monkeypatch.setenv("KLLM_ENGINE", "persistent")
    fast = Decoder(shape, w, numerics="fast")
    assert create_rc(lib, [fast]) == E_UNSUPPORTED
    assert create_rc(lib, [Decoder(shape, w, numerics="fast", kv_cache="bf16")]) == E_UNSUPPORTED
    hs64 = replace(GEOMETRIES["gqa-hs64"], seq_len=256)  # the fp8 cache takes head_size 64 and up
    assert create_rc(lib, [Decoder(hs64, synth_weights(hs64, "cuda", 4), numerics="fast", kv_cache="fp8")]) == \
        E_UNSUPPORTED
    if engine == "persistent":
        # another attention split at create: another cache layout
        split = a.attention_geometry[1]
        for v in ("1", "2", "4"):
            monkeypatch.setenv("KLLM_ATTN_SPLIT", v)
            c = Decoder(shape, w)
            if c.attention_geometry[1] != split:
                assert create_rc(lib, [a, c]) == E_UNSUPPORTED
                break
        else:
            pytest.fail("no KLLM_ATTN_SPLIT gave another split")
        monkeypatch.delenv("KLLM_ATTN_SPLIT")
    monkeypatch.setenv("KLLM_ENGINE", engine)
    batch = Batch([a, b])
    for tokens, pos, k in (([1, 2], [S - 4, 0], 5), ([1, V], [0, 0], 2), ([-1, 2], [0, 0], 2), ([1, 2], [-1, 0], 2),
                           ([1, 2], [0, 0], 0)):
        with pytest.raises(KllmError):
            batch.generate(tokens, pos, k)
    with pytest.raises(KllmError):
        batch.step([1, 2], [0, S])
    t2, p2, o2 = (ctypes.c_int32 * 2)(1, 2), (ctypes.c_int32 * 2)(0, 0), (ctypes.c_int32 * 2)()
    assert lib.kllm_batch_step(batch.handle, None, p2, o2) == E_INVALID
    assert lib.kllm_batch_step(batch.handle, t2, None, o2) == E_INVALID
    assert lib.kllm_batch_step(batch.handle, t2, p2, None) == E_INVALID
    assert lib.kllm_batch_step(None, t2, p2, o2) == E_INVALID
    assert lib.kllm_batch_generate(batch.handle, t2, p2, 1, None) == E_INVALID
    batch.close()
    for d, snap, name in ((a, snaps[0], "a"), (b, snaps[1], "b")):
        assert_unchanged(d, snap, f"member {name} after the refusals")


def assert_prefix_equal(a, b, n, what):
    assert np.array_equal(a.history()[:n], b.history()[:n]), f"{what}: history"
    for x, y in zip(a.logprobs(0, n), b.logprobs(0, n)):
        assert np.array_equal(np.asarray(x).view(np.uint32) if x.dtype == np.float32 else x,
                              np.asarray(y).view(np.uint32) if y.dtype == np.float32 else y), f"{what}: record"
    for x, y in zip(a.kv_cache(), b.kv_cache()):
        assert_bit_equal(x[:, :n], y[:, :n], f"{what}: kv rows")


@pytest.mark.parametrize("config", ["persistent", "graph", "fast-bf16", "fast-fp8"])
def test_copy_prefix(kllm_lib, monkeypatch, config):
    engine = "graph" if config == "graph" else "persistent"
    monkeypatch.setenv("KLLM_ENGINE", engine)
    # the fp8 cache takes head_size 64 and up
    shape = replace(GEOMETRIES["gqa-hs64"] if config == "fast-fp8" else SHAPES["small"], seq_len=256)
    w = synth_weights(shape, "cuda", 31)
    kw = {}
    if config.startswith("fast"):
        kv = config.split("-")[1]
        kw = dict(numerics="fast", kv_cache=kv)
        if kv == "fp8":
            rng = np.random.default_rng(3)
            kw["kv_scales"] = rng.uniform(0.01, 0.03, (2, shape.layer_num, shape.kv_head_num)).astype(np.float32)
    src, twin, dst = (Decoder(shape, w, **kw) for _ in range(3))
    assert dst.engine == engine
    for d in (src, twin, dst):
        d.set_logprobs(3)
    dst.set_sampling(0.9, 30, 5)  # dst keeps its own settings; the twin takes them after its prompt
    dst.generate(2, 0, 150)  # rows the copy overwrites, and rows past it
    prompt = [(5 * i + 2) % shape.vocab_size for i in range(70)]
    n = len(prompt) - 1
    src.prompt(prompt[:-1], 0), twin.prompt(prompt[:-1], 0)
    twin.set_sampling(0.9, 30, 5)
    dst.copy_prefix(src, n)
    assert_prefix_equal(dst, src, n, "after the copy")
    ids = dst.generate(prompt[-1], n, 20)
    assert twin.generate(prompt[-1], n, 20) == ids
    assert_bit_equal(dst.logits(), twin.logits(), "logits")
    assert_prefix_equal(dst, twin, n + 20, "after the copy and generate")
    # refusals copy nothing
    lib = dst.lib
    snap = snapshot(dst)
    other = Decoder(shape, synth_weights(shape, "cuda", 32), **kw)
    assert lib.kllm_decoder_copy_prefix(dst.handle, other.handle, 10) == E_UNSUPPORTED
    if config == "fast-fp8":
        kw2 = dict(kw, kv_scales=kw["kv_scales"] * 2)
        assert lib.kllm_decoder_copy_prefix(dst.handle, Decoder(shape, w, **kw2).handle, 10) == E_UNSUPPORTED
    for bad in (-1, shape.seq_len + 1):
        assert lib.kllm_decoder_copy_prefix(dst.handle, src.handle, bad) == E_INVALID
    assert lib.kllm_decoder_copy_prefix(dst.handle, dst.handle, 10) == E_INVALID
    assert lib.kllm_decoder_copy_prefix(None, src.handle, 10) == E_INVALID
    assert lib.kllm_decoder_copy_prefix(dst.handle, None, 10) == E_INVALID
    assert_unchanged(dst, snap, "dst after the refused copies")


def test_parallel_sampling_of_one_prompt(kllm_lib, engine):
    """One prompt prefilled once, copied into 7 decoders with other seeds and batched, against 8 decoders that each
    feed the prompt and generate on their own."""
    shape = replace(SHAPES["small"], seq_len=256)
    w = synth_weights(shape, "cuda", 8)
    try:
        ds = [Decoder(shape, w) for _ in range(2 * MAX_BATCH)]
    except KllmError:
        pytest.skip("engine")
    if ds[0].engine != engine:
        pytest.skip("engine")
    forks, refs = ds[:MAX_BATCH], ds[MAX_BATCH:]
    prompt = [(13 * i + 7) % shape.vocab_size for i in range(41)]
    n = len(prompt) - 1
    for d in ds:
        d.set_logprobs(2)
    forks[0].prompt(prompt[:-1], 0)
    for f in forks[1:]:
        f.copy_prefix(forks[0], n)
    for r in refs:
        r.prompt(prompt[:-1], 0)
    for b, (f, r) in enumerate(zip(forks, refs)):
        f.set_sampling(1.0, 50, 100 + b), r.set_sampling(1.0, 50, 100 + b)
    batch = Batch(forks)
    ids = batch.generate([prompt[-1]] * MAX_BATCH, [n] * MAX_BATCH, 30)
    batch.close()
    for b, r in enumerate(refs):
        assert r.generate(prompt[-1], n, 30) == ids[b], b
        assert_same_state(forks[b], r, n + 30, f"fork {b}")
    assert len({tuple(x) for x in ids}) > 1, "the seeds gave one continuation"
