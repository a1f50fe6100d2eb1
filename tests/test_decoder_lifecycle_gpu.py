"""-m gpu: decoders as real callers hold them, against the fp64 model of tests/prefill_model.py with the harness and
bounds of tests/decode_model_util.py.

Coexistence.  A speculative-decoding setup keeps a draft and a target decoder in one process, and a server may host
two models.  Each pair below is created one decoder after the other, then teacher-forced in interleaved segments
ending on each decoder's tile edges (A, B, A, B, ...); the second-created decoder is destroyed before the first one's
last segment.  Each decoder is held to its own fp64 model at every segment end and every K / V row, and bit for bit
to a solo run of the same decoder and segments.  Every pair runs in both creation orders.  The persistent engine's
kernels take a dynamic shared-memory size that is an attribute of the kernel function, one value per process, and
each decoder asks for its own (mega_smem_bytes): each pair differs in it, so one of the two orders creates the
larger decoder first and then launches it after the smaller one has configured the same kernel.

Rewind.  Chat regeneration, rejected draft tokens and prefix reuse feed a decoder from an earlier position again,
over cache rows an earlier, longer run left behind.  Sequence A is teacher-forced over all but the last position;
then sequence B, equal to A up to r and different after it, is fed from r to END_GAP positions before the end, for
every r of the geometry's edge_ends.  The first call after the rewind goes through one of the decoder's entry points
(step, generate, generate_until with the stop id mid-tile, prompt, the batched prefill, score), cycling over r; the
rest of B follows in teacher-forced segments.  The logits at each segment end and every row up to B's end are held
to the fp64 model of B; the logits, the rows and what the entry returned are bit for bit those of a fresh decoder
fed B in the same segments; and the rows past B's end still hold A's bits.

Measured worst values (an NVIDIA H100 80GB HBM3 at a 700 W power limit, 132 SMs) are printed with the [lifecycle]
tag; every case stays within the shared constants.  Worst err / bound over the module: coexistence, logits 0.379
(LOGIT_TAU), K / V 0.353 (KV_TAU); rewind, logits 0.358, K / V 0.365, the prefill's segment 0.469 and 0.564 (the
TF32 and bf16 prefill bounds), score's log-probabilities 0.0646; bf16 rows 0.998 of one ulp + KV_TAU rms.
"""
import ctypes
from dataclasses import replace

import numpy as np
import pytest
import torch

from decode_model_util import (GEOMETRIES, KV_TAU, KV_TAU_FIRST, LOGIT_TAU, WEIGHTS, device_sincos, edge_ends, fmt,
                               kv_ratios, logit_ratio, make_decoder, same_bits, sequence, stage_bytes)
from kv_bf16_model import bf16_rne, prefill_ref_bf16
from prefill_model import prefill_ref
from test_kv_bf16_gpu import ulp_bf16
from test_logprobs_gpu import check_entry
from test_prefill_tf32_model_gpu import KV_TAU as PREFILL_KV_TAU, LOGIT_TAU as PREFILL_LOGIT_TAU

from kuiperllama_b200 import ModelShape, sampling

pytestmark = pytest.mark.gpu

TAG = "[lifecycle]"


def report(*parts):
    print(TAG, *parts, flush=True)


# ---- the persistent engine's shared memory (MegaEngine::init) ----------------------------------------------------
DRAW_SCRATCH = 2592  # sampling::kDrawScratchBase
LOGPROB_SCRATCH = 5072  # sampling::logprob_scratch_bytes(256)
H100_SMEM_OPTIN = 227 * 1024  # cudaDevAttrMaxSharedMemoryPerBlockOptin


def mega_smem_bytes(shape, numerics, kv_cache="fp32", env=None, max_smem=H100_SMEM_OPTIN):
    """smem_bytes_ = xbuf + xres + stages * stage.  xbuf: the largest input row (max(dim, hidden, q rows) floats), the
    fast mode's flash partials and the draw and log-probability scratch, rounded up to 128; xres: dim floats, rounded
    up to 128; stages: as many as fit max_smem - xbuf - xres - 3584, at most 16.  Both rings fill that budget to
    within one stage, so the remainder decides which of two models asks for more."""
    env = env or {}
    fast = numerics == "fast"
    dim, hs = shape.dim, shape.head_size
    xbuf = max(max(dim, shape.hidden_dim, shape.head_num * hs) * 4, 2 * hs * 4)
    stage = stage_bytes(shape, numerics, env, kv_cache)
    if fast:
        xbuf = max(xbuf, (2 * hs + 8 * (hs + 2)) * 4)
    xbuf = (max(xbuf, DRAW_SCRATCH + 64 * 8, LOGPROB_SCRATCH) + 127) & ~127
    xres = (dim * 4 + 127) & ~127
    stages = min((max_smem - xbuf - xres - 3584) // stage, 16)
    return xbuf + xres + stages * stage


# ---- shapes ------------------------------------------------------------------------------------------------------
TINYLLAMA_2L = replace(GEOMETRIES["tinyllama-1.1b"], layer_num=2)
# The graph engine opts in above 48 KB for a gemv input row of more than 12288 floats (W2's, hidden_dim) and for an
# attention head wider than 188 (its q row and two 32-timestep value tiles): 56 KB and 65 KB, then 50 KB and 49 KB.
GRAPH_WIDE = ModelShape("graph-h14336-hs256", 512, 14336, 2, 2, 2, 4096, 544)
GRAPH_NARROW = ModelShape("graph-h12800-hs192", 384, 12800, 2, 2, 1, 4096, 544)
SHAPES_BY_KEY = {"tinyllama-2l": TINYLLAMA_2L, "small": GEOMETRIES["small"], "hs128": GEOMETRIES["hs128"],
                 "small-int8": GEOMETRIES["small-int8"], "llama2-7b-int8-2l": GEOMETRIES["llama2-7b-int8-2l"],
                 "graph-wide": GRAPH_WIDE, "graph-narrow": GRAPH_NARROW}


# ---- models held side by side -----------------------------------------------------------------------------------
_MODELS = {}


@pytest.fixture(scope="module")
def models(kllm_lib):
    """get(key, weights, kind) -> (shape, weights, tokens, model) with kind "plain" or "fixed" (the fast mode's
    fixed-point rule, int8 group 64), the model's logits at every position; every model of the module is kept, so
    that both decoders of a pair have theirs at once."""
    def get(key, weights, kind):
        ck = (key, weights, kind)
        if ck not in _MODELS:
            shape = SHAPES_BY_KEY[key]
            wk = (key, weights)
            if wk not in _MODELS:
                _MODELS[wk] = WEIGHTS[weights](shape, "cuda", 77)
            w = _MODELS[wk]
            toks = sequence(shape.vocab_size, shape.seq_len, 5)
            sin, cos = device_sincos(kllm_lib, shape)
            _MODELS[ck] = (shape, w, toks, prefill_ref(w, shape, toks, 0, sin, cos, tf32=False,
                                                       logits_at=range(shape.seq_len),
                                                       fixed_point=kind == "fixed"))
        return _MODELS[ck]
    yield get
    _MODELS.clear()
    torch.cuda.empty_cache()


# ---- coexisting decoders -----------------------------------------------------------------------------------------
# side: (shape key, weights, numerics, engine, kv cache, env).  The persistent engine's smem_bytes_ of each side on an
# H100 (227 KB opt-in), as mega_smem_bytes computes it from MegaEngine::init's rule; the test asserts they differ:
#   tinyllama-2l exact 227328, fast 227328, bf16 227328   small exact 202880, fast 219264, bf16 202880
#   llama2-7b-int8-2l fast 226304                          small-int8 fast 227328 (the small model asks for more)
#   hs128 exact 204160
# The graph pair differs in the gemv and attention opt-ins above.
TL = "tinyllama-2l"
PAIRS = {
    # kllm_decoder_profile on the older decoder runs the profiling instantiation after the younger one's init
    "fp32-exact": ((TL, "synth", "exact", "persistent", "fp32", {}),
                   ("small", "synth", "exact", "persistent", "fp32", {}), {"profile": True}),
    # set_logprobs(5) on both: the log-probability instantiation
    "fp32-fast-logprobs": ((TL, "synth", "fast", "persistent", "fp32", {}),
                           ("small", "synth", "fast", "persistent", "fp32", {}), {"logprobs": 5}),
    "int8-fast": (("llama2-7b-int8-2l", "outliers", "fast", "persistent", "fp32", {}),
                  ("small-int8", "outliers", "fast", "persistent", "fp32", {}), {}),
    "bf16": ((TL, "synth", "fast", "persistent", "bf16", {}),
             ("small", "synth", "fast", "persistent", "bf16", {}), {}),
    "streams": (("small", "loud", "exact", "persistent", "fp32", {}),
                ("hs128", "loud", "exact", "persistent", "fp32", {}), {"streams": True}),
    "graph": (("graph-wide", "loud", "exact", "graph", "fp32", {}),
              ("graph-narrow", "loud", "exact", "graph", "fp32", {}), {}),
    "mixed": ((TL, "synth", "exact", "persistent", "fp32", {}),
              ("graph-narrow", "loud", "exact", "graph", "fp32", {}), {}),
}
PAIR_CASES = [(name, order) for name in PAIRS for order in ("ab", "ba")]


def model_kind(side):
    key, _, numerics, _, kv_cache, _ = side
    return "fixed" if numerics == "fast" and SHAPES_BY_KEY[key].group_size == 64 else "plain"


def side_ends(dec, shape):
    if dec.engine == "persistent":
        T, SP = dec.attention_geometry[:2]
    else:
        T, SP = 32, 1  # mha_decode_kernel's value tile
    return edge_ends(T, SP, shape.seq_len)


class Side:
    """One decoder of a pair, run segment by segment; records the logits at every end and the log-probability
    record of every segment."""

    def __init__(self, monkeypatch, models, side, stream=None, top_n=-1):
        key, weights, numerics, engine, kv_cache, env = side
        self.what = f"{key} {numerics} {engine} {kv_cache}"
        self.shape, self.w, self.toks, self.model = models(key, weights, model_kind(side))
        self.kv_cache = kv_cache
        self.dec = make_decoder(monkeypatch, self.shape, self.w, numerics, env, engine=engine, kv_cache=kv_cache)
        self.stream = stream
        if stream is not None:  # make_decoder builds on the default stream; a caller stream is the Decoder's own
            self.dec.close()
            self.dec = _decoder_on(self.shape, self.w, numerics, kv_cache, stream)
        self.top_n = top_n
        if top_n >= 0:
            self.dec.set_logprobs(top_n)
        self.ends = side_ends(self.dec, self.shape)
        self.start, self.logits, self.records, self.ids = 0, {}, {}, {}

    def segment(self, i):
        end = self.ends[i]
        assert self.start <= end
        self.ids[end] = self.dec.generate(0, self.start, end + 1 - self.start,
                                          teacher=self.toks[self.start:end + 1])
        self.logits[end] = self.dec.logits()
        if self.top_n >= 0:
            self.records[end] = self.dec.logprobs(self.start, end + 1 - self.start)
        self.start = end + 1

    def finish(self):
        self.kv = self.dec.kv_cache()


def _decoder_on(shape, w, numerics, kv_cache, stream):
    from kuiperllama_b200 import Decoder
    return Decoder(shape, w, stream=stream, numerics=numerics, kv_cache=kv_cache)


def check_side_against_model(kllm_lib, s):
    """Logits at every end and every K / V row against the side's fp64 model (the bf16 cache: the bf16 model fed
    the decoder's own rows, test_kv_bf16_gpu.py's bounds); returns the worst ratios."""
    shape, ref = s.shape, s.model
    worst_logit = 0.0
    if s.kv_cache == "bf16":
        sin, cos = device_sincos(kllm_lib, shape)
        k, v = (torch.from_numpy(a).cuda() for a in s.kv)
        ref = prefill_ref_bf16(s.w, shape, s.toks, 0, sin, cos, tf32=False, logits_at=s.ends,
                               fixed_point=shape.group_size == 64, rule="decode", kv_rows=(k, v))
        worst_kv = 0.0
        for name, got, r in (("K", k, ref["k"]), ("V", v, ref["v"])):
            assert torch.equal(bf16_rne(got), got.float()), (s.what, name)
            want = bf16_rne(r).double()
            bound = ulp_bf16(want) + KV_TAU * r.pow(2).mean(-1, keepdim=True).sqrt()
            worst_kv = max(worst_kv, float(((got.double() - want).abs() / bound).max()))
        per_layer = {"K / V vs ulp + KV_TAU rms": [worst_kv]}
    else:
        per_layer = kv_ratios(s.kv, ref, KV_TAU, KV_TAU_FIRST)
    for end in s.ends:
        lref = ref["logits_at"][end]
        worst_logit = max(worst_logit, logit_ratio(s.logits[end], lref, LOGIT_TAU))
        bound = LOGIT_TAU * float(lref.pow(2).mean().sqrt())
        top2 = torch.topk(lref, 2).values
        if float(top2[0] - top2[1]) > 2 * bound:
            assert s.ids[end][-1] == int(torch.argmax(lref)), (s.what, end)
        if s.top_n >= 0:
            rid, rlp, rtop, rtop_lp = (a[-1] for a in s.records[end])
            assert rid == s.ids[end][-1], (s.what, end)
            check_entry(s.logits[end], shape.vocab_size, rid, rlp, rtop, rtop_lp, s.top_n, (s.what, end))
    assert worst_logit <= 1.0, (s.what, worst_logit)
    for name, v in per_layer.items():
        assert max(v) <= 1.0, (s.what, name, v)
    return worst_logit, per_layer


def compare_runs(what, a, b):
    for end in a.ends:
        assert a.ids[end] == b.ids[end], (what, "ids", end)
        assert same_bits(a.logits[end], b.logits[end]), (what, "logits", end)
        for x, y in zip(a.records.get(end, ()), b.records.get(end, ())):
            assert same_bits(x, y), (what, "log-probability record", end)
    for name, x, y in (("K", a.kv[0], b.kv[0]), ("V", a.kv[1], b.kv[1])):
        assert same_bits(x, y), (what, name)


def profile_once(dec):
    """One kllm_decoder_profile call of two steps from position 0 (the profiling instantiation); its return code."""
    lib = dec.lib
    grid, phases = ctypes.c_int32(0), ctypes.c_int32(0)
    probe = np.zeros(1, np.uint64)
    lib.kllm_decoder_profile(dec.handle, 1, 0, 2, 1, probe.ctypes.data_as(ctypes.c_void_p), 0, ctypes.byref(grid),
                             ctypes.byref(phases))
    buf = np.zeros(grid.value * phases.value * 16, np.uint64)  # kProfStamps stamps per CTA and phase
    return lib.kllm_decoder_profile(dec.handle, 1, 0, 2, 1, buf.ctypes.data_as(ctypes.c_void_p), buf.size,
                                    ctypes.byref(grid), ctypes.byref(phases))


@pytest.mark.parametrize("name,order", PAIR_CASES, ids=[f"{n}-{o}" for n, o in PAIR_CASES])
def test_coexisting_decoders(kllm_lib, monkeypatch, models, name, order):
    first, second, opts = PAIRS[name]
    if order == "ba":
        first, second = second, first
    persistent = [s for s in (first, second) if s[3] == "persistent"]
    if len(persistent) == 2:
        sizes = [mega_smem_bytes(SHAPES_BY_KEY[s[0]], s[2], s[4], s[5]) for s in persistent]
        assert sizes[0] != sizes[1], (name, sizes)
    top_n = opts.get("logprobs", -1)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()] if opts.get("streams") else [None, None]
    handles = [st.cuda_stream if st is not None else None for st in streams]

    a = Side(monkeypatch, models, first, handles[0], top_n)
    b = Side(monkeypatch, models, second, handles[1], top_n)
    # A, B, A, B, ...; A's last segment after B is destroyed
    for i in range(max(len(a.ends) - 1, len(b.ends))):
        if i < len(a.ends) - 1:
            a.segment(i)
        if i < len(b.ends):
            b.segment(i)
    b.finish()
    b.dec.close()
    a.segment(len(a.ends) - 1)
    a.finish()
    if opts.get("profile"):
        assert profile_once(a.dec) == 0, name
    a.dec.close()

    for s, side, h in ((a, first, handles[0]), (b, second, handles[1])):
        solo = Side(monkeypatch, models, side, h, top_n)
        for i in range(len(solo.ends)):
            solo.segment(i)
        solo.finish()
        solo.dec.close()
        compare_runs(f"{name} {order}: {s.what} beside the other decoder vs solo", s, solo)
        worst_logit, per_layer = check_side_against_model(kllm_lib, s)
        report(f"{name} {order}: {s.what} ({len(s.ends)} segments, bit for bit its solo run): logits err / bound "
               f"{worst_logit:.3g}; K / V err / bound per layer {fmt(per_layer)}")


# ---- rewind and reuse --------------------------------------------------------------------------------------------
END_GAP = 12  # B ends END_GAP positions before A's last row: rows past B's end must keep A's bits
REWIND_GEOMETRIES = {
    "small": (replace(GEOMETRIES["small"], seq_len=1056), "loud"),
    "hs128": (GEOMETRIES["hs128"], "loud"),
    "small-int8": (GEOMETRIES["small-int8"], "outliers"),
    "qwen2.5-reduced": (replace(GEOMETRIES["qwen2.5-reduced"], seq_len=2080), "synth"),
}


def t32_stage(shape):
    return str(32 * shape.head_size * 4)


# config -> (numerics, engine, kv cache, env of the shape)
CONFIGS = {
    "exact": ("exact", "persistent", "fp32", lambda s: {}),  # hs128: split 8, V slices and tagged scores
    "fast": ("fast", "persistent", "fp32", lambda s: {}),
    "fast-sp8-t32": ("fast", "persistent", "fp32", lambda s: {"KLLM_ATTN_SPLIT": "8", "KLLM_STAGE_BYTES": t32_stage(s)}),
    "bf16": ("fast", "persistent", "bf16", lambda s: {}),
    "graph": ("exact", "graph", "fp32", lambda s: {}),
}
ENTRIES = ["generate", "step", "generate_until", "prompt", "prefill", "score"]


@pytest.fixture(scope="module", params=list(REWIND_GEOMETRIES))
def rewind_geometry(request, kllm_lib):
    """(key, shape, weights, A, C, sin, cos, {kind: A's model rows}); B_r = A[:r] + C[r:]."""
    key = request.param
    shape, weights = REWIND_GEOMETRIES[key]
    _MODELS.clear()
    torch.cuda.empty_cache()
    w = WEIGHTS[weights](shape, "cuda", 77)
    A = sequence(shape.vocab_size, shape.seq_len, 5)
    C = sequence(shape.vocab_size, shape.seq_len, 6)
    sin, cos = device_sincos(kllm_lib, shape)
    n_a = shape.seq_len - 1
    rows = {}
    for kind in ("plain", "fixed") if shape.group_size == 64 else ("plain",):
        m = prefill_ref(w, shape, A[:n_a], 0, sin, cos, tf32=False, fixed_point=kind == "fixed")
        rows[kind] = (m["k"], m["v"])
    yield key, shape, w, A, C, sin, cos, rows
    torch.cuda.empty_cache()


class Feed:
    """B fed from r through one entry point, then in teacher-forced segments to `end_b`; records what each call
    returned and the logits at each segment end."""

    def __init__(self, entry, r, ends, B, T, seed):
        self.entry, self.r, self.ends, self.B, self.T, self.seed = entry, r, ends, B, T, seed
        self.stop = None

    def run(self, dec):
        r, B, ends = self.r, self.B, self.ends
        out, logits = [], {}
        start = r
        for i, end in enumerate(ends):
            toks = B[start:end + 1]
            if i > 0 or self.entry == "generate":
                out.append(dec.generate(0, start, len(toks), teacher=toks))
            elif self.entry == "step":
                out.append(dec.step(toks[0], start))
            elif self.entry == "prompt":
                out.append(dec.prompt(toks, start))
            elif self.entry == "prefill":
                out.append(dec.prefill_w8(toks, start) if dec.shape.group_size else dec.prefill_tf32(toks, start))
            elif self.entry == "score":
                # feeds toks[:-1]; toks[-1] continues the sequence at `end`
                out.append(dec.score(toks, start).view(np.uint32).tolist())
                out.append(dec.step(toks[-1], end))
            elif self.entry == "generate_until":
                dec.set_sampling(1.0, 0, self.seed)
                room = min(len(toks) + self.T, dec.shape.seq_len - start)  # the stop id, not max_steps, ends it
                out.append(dec.generate_until(toks[0], start, room, stop_ids=[self.stop]))
                dec.set_sampling(0.0)
                assert out[-1][-1] == self.stop and len(out[-1]) == len(toks), (out[-1], self.stop)
            logits[end] = dec.logits()
            start = end + 1
        return out, logits


def entry_ends(entry, r, ends_all, end_b):
    """The segment ends of B from r: the first one is the entry's call (one position for step, B up to end_b for
    score)."""
    if entry == "step":
        return [r] + [e for e in ends_all if r < e < end_b] + [end_b]
    if entry == "score":
        return [end_b]
    return [e for e in ends_all if r <= e < end_b] + [end_b]


def sampled_stop(dec, feed, B, r, T, max_steps):
    """generate_until's sampled continuation from r (seeded: the ids depend only on the seed, the position and the
    logits) on a fresh decoder fed B[:r]; the stop id is the first id that appears for the first time at or after the
    middle of the tile after r's, and B's ids from r + 1 become the sampled ones up to it."""
    if r:
        dec.generate(0, 0, r, teacher=B[:r])
    dec.set_sampling(1.0, 0, feed.seed)
    ids = dec.generate_until(B[r], r, max_steps)
    dec.set_sampling(0.0)
    target = min((r // T + 1) * T + T // 2 - r, max_steps - 1)
    order = list(range(target, max_steps)) + list(range(target - 1, -1, -1))
    k = next(i for i in order if ids[i] not in ids[:i])
    return ids[k], B[:r + 1] + [int(t) for t in ids[:k]] + B[r + k + 1:], r + k


def test_rewind_against_the_model_and_a_fresh_decoder(kllm_lib, monkeypatch, rewind_geometry, config):
    key, shape, w, A, C, sin, cos, a_rows = rewind_geometry
    numerics, engine, kv_cache, env_of = CONFIGS[config]
    env = env_of(shape)
    fixed = numerics == "fast" and shape.group_size == 64
    kind = "fixed" if fixed else "plain"

    def new():
        return make_decoder(monkeypatch, shape, w, numerics, env, engine=engine, kv_cache=kv_cache)

    dec = new()
    T, SP = dec.attention_geometry[:2] if engine == "persistent" else (32, 1)
    n_a = shape.seq_len - 1
    end_b = n_a - 1 - END_GAP
    ends_all = edge_ends(T, SP, shape.seq_len)
    rs = [e for e in ends_all if e < end_b]
    worst = {"logits": 0.0, "kv": 0.0, "prefill logits": 0.0, "prefill kv": 0.0, "score lp": 0.0}
    seen = []
    for i, r in enumerate(rs):
        entry = ENTRIES[(i + list(CONFIGS).index(config)) % len(ENTRIES)]
        B = A[:r] + C[r:]
        ends = entry_ends(entry, r, ends_all, end_b)
        feed = Feed(entry, r, ends, B, T, seed=1000 + r)
        if entry == "generate_until":
            probe = new()
            feed.stop, B, until_end = sampled_stop(probe, feed, B, r, T, min(2 * T, end_b + 1 - r))
            probe.close()
            ends = [until_end] + [e for e in ends if e > until_end]
            feed.ends, feed.B = ends, B
        what = f"{key} {config} r={r} {entry}"

        # the rewound decoder: A over all but the last position, then B from r
        dec.generate(0, 0, n_a, teacher=A[:n_a])
        if i == 0:
            k_a, v_a = dec.kv_cache()
        got, logits = feed.run(dec)
        k, v = dec.kv_cache()
        assert same_bits(k[:, end_b + 1:], k_a[:, end_b + 1:]) and same_bits(v[:, end_b + 1:], v_a[:, end_b + 1:]), \
            (what, "rows past B's end")

        # a fresh decoder fed B[:r], then the same calls
        fresh = new()
        if r:
            fresh.generate(0, 0, r, teacher=B[:r])
        got_f, logits_f = feed.run(fresh)
        k_f, v_f = fresh.kv_cache()
        fresh.close()
        assert got == got_f, what
        for end in ends:
            assert same_bits(logits[end], logits_f[end]), (what, "logits", end)
        assert same_bits(k[:, :end_b + 1], k_f[:, :end_b + 1]) and same_bits(v[:, :end_b + 1], v_f[:, :end_b + 1]), \
            (what, "rows up to B's end")

        check_rewind_against_the_model(what, kllm_lib, shape, w, B, r, ends, end_b, (k, v), logits, got, entry,
                                       a_rows[kind], sin, cos, fixed, kv_cache, worst)
        seen.append(f"{r}:{entry}")
    dec.close()
    report(f"{key} {config} T={T} SP={SP}: rewinds {seen}, each bit for bit a fresh decoder; worst err / bound "
           f"{ {k: float(f'{v:.3g}') for k, v in worst.items()} }")


def check_rewind_against_the_model(what, kllm_lib, shape, w, B, r, ends, end_b, kv, logits, got, entry, a_rows, sin,
                                   cos, fixed, kv_cache, worst):
    k, v = (torch.from_numpy(x).cuda() for x in kv)
    start = r
    if entry == "prefill":  # the prefill's segment against the TF32 model over the rows before r
        e1 = ends[0]
        kv_in = (k[:, :r], v[:, :r]) if kv_cache == "bf16" else a_rows
        n = e1 + 1 - r
        if kv_cache == "bf16":
            ref = prefill_ref_bf16(w, shape, B[r:e1 + 1], r, sin, cos, rule="prefill", tf32=True, kv_in=kv_in,
                                   logits_at=[n - 1])
        else:
            ref = prefill_ref(w, shape, B[r:e1 + 1], r, sin, cos, kv_in=kv_in, tf32=True, logits_at=[n - 1])
        lref = ref["logits_at"][n - 1]
        bound = (2e-2 * float(lref.abs().max()) if kv_cache == "bf16"
                 else PREFILL_LOGIT_TAU * float(lref.pow(2).mean().sqrt()))
        ratio = float((torch.from_numpy(logits[e1]).cuda().double() - lref).abs().max()) / bound
        worst["prefill logits"] = max(worst["prefill logits"], ratio)
        assert ratio <= 1.0, (what, "prefill logits", ratio)
        for name, g, exp in (("K", k[:, r:e1 + 1], ref["k"]), ("V", v[:, r:e1 + 1], ref["v"])):
            rms = exp.pow(2).mean(-1, keepdim=True).sqrt()
            if kv_cache == "bf16":
                want = bf16_rne(exp).double()
                b = ulp_bf16(want) + (5e-2 if shape.group_size else 1e-2) * (rms + 1e-3)
            else:
                want, b = exp, PREFILL_KV_TAU * rms
            ratio = float(((g.double() - want).abs() / b).max())
            worst["prefill kv"] = max(worst["prefill kv"], ratio)
            assert ratio <= 1.0, (what, "prefill", name, ratio)
        start, ends = e1 + 1, ends[1:]
        if not ends:
            return
    # decode positions start .. end_b: over the model's rows before r, or, after the prefill's segment, over the
    # decoder's own rows (its TF32 error does not count against the decode bounds); a bf16 cache feeds the model
    # the decoder's rows
    if kv_cache == "bf16" or start > r:
        kv_in = (k[:, :start], v[:, :start])
    else:
        kv_in = a_rows
    rel = [e - start for e in ends]
    toks = B[start:end_b + 1]
    lp_at = range(len(toks)) if entry == "score" else rel
    if kv_cache == "bf16":
        ref = prefill_ref_bf16(w, shape, toks, start, sin, cos, rule="decode", kv_in=kv_in,
                               kv_rows=(k[:, start:], v[:, start:]), tf32=False, logits_at=lp_at, fixed_point=fixed)
    else:
        ref = prefill_ref(w, shape, toks, start, sin, cos, kv_in=kv_in, tf32=False, logits_at=lp_at,
                          fixed_point=fixed)
    for e, re_ in zip(ends, rel):
        worst["logits"] = max(worst["logits"], logit_ratio(logits[e], ref["logits_at"][re_], LOGIT_TAU))
    assert worst["logits"] <= 1.0, (what, "logits", worst["logits"])
    got_rows = (k[:, start:end_b + 1], v[:, start:end_b + 1])
    if kv_cache == "bf16":
        for name, g, r_ in (("K", got_rows[0], ref["k"]), ("V", got_rows[1], ref["v"])):
            want = bf16_rne(r_).double()
            bound = ulp_bf16(want) + KV_TAU * r_.pow(2).mean(-1, keepdim=True).sqrt()
            worst["kv"] = max(worst["kv"], float(((g.double() - want).abs() / bound).max()))
    else:
        per_layer = kv_ratios(tuple(x.cpu().numpy() for x in got_rows), ref, KV_TAU, KV_TAU_FIRST)
        worst["kv"] = max([worst["kv"]] + [max(x) for x in per_layer.values()])
    assert worst["kv"] <= 1.0, (what, "K / V", worst["kv"])
    if entry == "score":  # lp[i] = log p(B[r + i + 1]) against the model's logits at r + i
        lp = np.asarray(got[0], np.uint32).view(np.float32)
        V = shape.vocab_size
        for i in range(len(lp)):
            lref = ref["logits_at"][i]
            lp64 = float(torch.log_softmax(lref, 0)[B[r + i + 1]])
            bound = 2 * LOGIT_TAU * float(lref.pow(2).mean().sqrt()) + float(sampling.logprob_bound(lp64, V, V))
            worst["score lp"] = max(worst["score lp"], abs(float(lp[i]) - lp64) / bound)
        assert worst["score lp"] <= 1.0, (what, "score", worst["score lp"])


@pytest.fixture(params=list(CONFIGS))
def config(request):
    return request.param
