"""The decode-step model harness shared by test_decode_model_gpu.py (the persistent engine, both numerics modes)
and test_graph_engine_model_gpu.py (the graph engine, and both engines at other int8 group sizes): weight
builders, the persistent engine's flash geometry, the seeded teacher sequence, one cached fp64 model at a time,
and `run`, which teacher-forces a decoder over every position and holds its logits and K / V rows to the model.

Bounds: each K / V element within KV_TAU * rms(row), the logits within LOGIT_TAU * rms(logits), and the greedy id
equal to the model's argmax wherever the model's top-2 margin exceeds twice the logit bound.  The constants and
their measured worst values are those of test_decode_model_gpu.py's docstring (an NVIDIA H100 80GB HBM3 at a 700 W
power limit; worst error / rms, exact mode then fast mode; both within 2x, so one constant serves both).
"""
import math
from dataclasses import replace

import numpy as np
import torch

from gpu_util import ptr, sync
from prefill_model import prefill_ref

from kuiperllama_b200 import FLAVOURS, SHAPES, Decoder, ModelShape, synth_weights
from kuiperllama_b200.decoder import quantize_q80

KV_TAU_FIRST = 1e-5  # layer 0 of every case: 2.47e-6, 2.43e-6
KV_TAU = 6e-5  # layers 1 and 2: 2.51e-5, 1.39e-5
LOGIT_TAU = 8e-5  # 2.57e-5, 2.08e-5
# TinyLlama-1.1B, 22 layers (synth weights: smaller errors than the loud 2 to 3 layer cases)
KV_TAU_DEEP = 2e-5  # layers 1 .. 21: 6.32e-6, 5.24e-6
LOGIT_TAU_DEEP = 2e-5  # 5.88e-6, 4.94e-6

KNOBS = ("KLLM_ENGINE", "KLLM_MODE", "KLLM_ATTN_SPLIT", "KLLM_STAGE_BYTES")


def report(*parts, tag="[decode-model]"):
    print(tag, *parts, flush=True)


# ---- weights --------------------------------------------------------------------------------------------------
def loud_weights(shape, device, seed):
    """synth_weights with wq and wk scaled so that q.k / sqrt(hs) has std ~5 (q and k elements of std sqrt(5) for
    unit-rms inputs) and Wo at std 1/sqrt(dim)."""
    w = synth_weights(shape, device, seed)
    c = math.sqrt(5.0 / (0.02 ** 2 * shape.dim))
    w["wq"] *= c
    w["wk"] *= c
    g = torch.Generator(device=device).manual_seed(seed + 1)
    w["wo"] = torch.empty_like(w["wo"]).normal_(0.0, 1.0 / math.sqrt(shape.dim), generator=g)
    return w


OUTLIER_CHANNELS = (5, -7)  # in the first and the last 64-group
ZERO_GROUP = slice(64, 128)  # the second 64-group


def outlier_weights(shape, device, seed):
    """int8 weights with massive activations and all-zero groups, built in fp32 and quantised as export.py does:
    two embedding channels at 300x the others (they dominate the residual stream of every layer), attn_norm zero on
    one 64-group (an all-zero group reaches the quantiser in the QKV phase) and W1 zero on 64 rows (the SwiGLU
    output, W2's input, is zero on that group), and weight bytes of -128 (the file format allows them; export.py
    never writes them) in every matrix."""
    w = synth_weights(replace(shape, group_size=0), device, seed)
    for c in OUTLIER_CHANNELS:
        w["tok_emb"][:, c] *= 300.0
    w["attn_norm"][:, ZERO_GROUP] = 0.0
    w["w1"][:, ZERO_GROUP, :] = 0.0
    g = torch.Generator(device=device).manual_seed(seed + 2)
    for name in ("wq", "wk", "wv", "wo", "w1", "w2", "w3", "wcls"):
        mats = [w[name]] if name == "wcls" else list(w[name])
        qs = [quantize_q80(t, shape.group_size) for t in mats]
        q = torch.stack([a for a, _ in qs])
        sc = torch.stack([b for _, b in qs])
        flat = q.view(-1)
        idx = torch.randint(0, flat.numel(), (64,), device=device, generator=g)
        flat[idx] = -128
        if name == "wcls":
            q, sc = q[0], sc[0]
        w[name], w["s" + name[1:]] = q.contiguous(), sc.contiguous()
    return w


WEIGHTS = {"synth": lambda shape, device, seed: synth_weights(shape, device, seed),
           "loud": loud_weights, "outliers": outlier_weights}


# ---- the persistent engine's attention geometry (MegaEngine::init) -----------------------------------------------
KV_ELEM_BYTES = {"fp32": 4, "bf16": 2, "fp8": 1}


def weight_format_of(shape, weight_format="fp32"):
    """The decoder's weight format: "int8" for a shape with an int8 group size, else the one asked for (fp32 or the
    bf16 weights of decoder.bf16_weights)."""
    assert weight_format in ("fp32", "bf16") or (weight_format == "int8" and shape.group_size), weight_format
    return "int8" if shape.group_size else weight_format


def stage_bytes(shape, numerics, env, kv_cache="fp32", weight_format="fp32"):
    """The ring stage MegaEngine::init picks: KLLM_STAGE_BYTES, else 27 KB for int8 weights, 24 KB for bf16 weights in
    the fast mode and 32 KB in the exact mode, 16 KB for fp32 weights in the fast mode with an fp32 cache when two input
    rows of dim fit (dim <= 2048), else 32 KB; rounded up to 128 bytes."""
    wf = weight_format_of(shape, weight_format)
    fast = numerics == "fast"
    if wf == "int8":
        default = 27 * 1024
    elif wf == "bf16":
        default = 24 * 1024 if fast else 32 * 1024
    else:
        default = 16 * 1024 if fast and kv_cache == "fp32" and 2 * shape.dim * 4 <= 16 * 1024 else 32 * 1024
    return (int(env.get("KLLM_STAGE_BYTES", default)) + 127) & ~127


def engine_geometry(shape, numerics, env, sms, kv_cache="fp32", weight_format="fp32"):
    """(tile T, split SP, V tile, stage bytes) the persistent engine chooses, which Decoder.attention_geometry
    reports; every persistent case asserts the two agree, so that a change to the rules fails loudly instead of
    moving the segment ends off the tiles' edges.
    Stage: stage_bytes.  T = min(stage / (hs * elem), 256) & ~31, elem the cache's element: 4 bytes for fp32, 2 for
    bf16, 1 for fp8.
    Split: the largest power of two <= 8 with heads * SP <= grid and, in the fast mode, SP * (hs + 2) <= seq_len, in
    the exact mode hs / SP a multiple of 4 (the exact mode splits only head sizes >= 128 unless asked); a
    KLLM_ATTN_SPLIT power of two up to that cap replaces it.  V tile: stage / ((hs / SP) * elem) & ~31 in the exact
    mode (V slices of hs / SP dims), stage / (hs * elem) & ~31 in the fast mode."""
    fast = numerics == "fast"
    hs = shape.head_size
    stage = stage_bytes(shape, numerics, env, kv_cache, weight_format)
    esz = KV_ELEM_BYTES[kv_cache]
    T = min(stage // (hs * esz), 8 * 32) & ~31
    grid = min(sms, shape.dim, shape.hidden_dim)
    cap = 1
    while cap * 2 <= 8 and shape.head_num * cap * 2 <= grid and (
            cap * 2 * (hs + 2) <= shape.seq_len if fast else (hs // (cap * 2)) % 4 == 0 and hs % (cap * 2) == 0):
        cap *= 2
    sp = cap if fast or hs >= 128 else 1
    asked = int(env.get("KLLM_ATTN_SPLIT", 0))
    if 1 <= asked <= cap and (asked & (asked - 1)) == 0:
        sp = asked
    T_v = (stage // ((hs // (1 if fast else sp)) * esz)) & ~31
    return T, sp, T_v, stage


def flash_geometry(shape, env, sms):
    """(tile T, split SP) of the fast mode with an fp32 cache under `env` (engine_geometry)."""
    return engine_geometry(shape, "fast", env, sms)[:2]


def split_cap(shape, sms):
    return flash_geometry(shape, {"KLLM_ATTN_SPLIT": "8"}, sms)[1]


def edge_ends(T, SP, seq_len):
    """Segment ends: the first blocks of 8 timesteps, the first tile's edge, the first CTA's second tile, the end."""
    e = {0, 1, 7, 8, 9, T - 1, T, T + 1, SP * T - 1, SP * T, SP * T + 1, seq_len - 1}
    return sorted(p for p in e if 0 <= p < seq_len)


def continue_ends(T, n, seq_len):
    """Segment ends of a decode that continues at position n (after a prefill of n rows) across the next edge of its
    T-timestep tiles."""
    edge = (n // T + 1) * T
    ends = sorted(p for p in {n, n + 1, edge - 1, edge, edge + 1} if n <= p < seq_len)
    assert ends[-1] >= edge, (T, n, seq_len)
    return ends


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- the persistent engine's cases (test_decode_model_gpu.py), which the graph engine repeats ---------------
# The flash tile T of the fast mode's default 16 KB stages (fp32 up to dim 2048; engine_geometry) and 27 KB (int8)
GEOMETRIES = {
    # dim 64, 4 / 2 heads: head_size 16, T = 256, 8 CTAs per head
    "hs16": ModelShape("decode-hs16", 64, 172, 2, 4, 2, 512, 2080),
    "small": replace(SHAPES["small"], seq_len=2080),  # head_size 32, GQA 3, T = 128
    "small-hs48": replace(SHAPES["small-hs48"], seq_len=1312),  # T = 64
    "hs128": ModelShape("decode-hs128", 512, 1376, 2, 4, 2, 2048, 1056),  # T = 32
    "small-qwen": replace(SHAPES["small-qwen"], seq_len=1056),  # bias, half-split pairs, eps 1e-6, T = 64
    # Llama-3-8B attention geometry and vocabulary at two layers: half-split pairs, theta 5e5; 32 KB stages, T = 64
    "llama3-reduced": ModelShape("llama3-reduced", 4096, 14336, 2, 32, 8, 128256, 544, flavour="llama3"),
    "small-int8": replace(SHAPES["small-int8"], seq_len=800),  # T = 96
    "small-tp-int8": replace(SHAPES["small-tp-int8"], seq_len=800),
    # Llama-2-7B int8 at two layers: T = 32, 4 CTAs per head
    "llama2-7b-int8-2l": replace(SHAPES["llama2-7b-int8"], layer_num=2, seq_len=544),
    "qwen2.5-reduced": ModelShape("qwen2.5-reduced", 896, 4864, 2, 14, 2, 4096, 16384, True,
                                  flavour="qwen2"),  # T = 64
    "tinyllama-1.1b": replace(SHAPES["tinyllama-1.1b"], seq_len=1024),  # T = 64
    # head_size 64, four query heads per KV head: the smallest head the fp8 cache's tile mapping takes (one 16-byte K
    # chunk per lane quarter); the reduced-precision caches' cases only
    "gqa-hs64": ModelShape("decode-gqa-hs64", 256, 688, 2, 4, 1, 1024, 1100),
}
# (geometry, weights, environment of the fast mode)
CASES = [("hs16", "loud", {}), ("small", "synth", {}), ("small", "loud", {}), ("small-hs48", "loud", {}),
         ("hs128", "loud", {}), ("small-qwen", "loud", {}), ("llama3-reduced", "loud", {}),
         ("small-int8", "synth", {}), ("small-int8", "outliers", {}), ("small-tp-int8", "synth", {}),
         ("llama2-7b-int8-2l", "outliers", {}),
         ("qwen2.5-reduced", "synth", {}), ("tinyllama-1.1b", "synth", {})]


def case_id(c):
    return "-".join([c[0], c[1]] + [f"{k[5:].lower()}{v}" for k, v in c[2].items()])


def taus(key):
    return (KV_TAU_DEEP, LOGIT_TAU_DEEP) if key == "tinyllama-1.1b" else (KV_TAU, LOGIT_TAU)


# ---- the model -----------------------------------------------------------------------------------------------------
def device_sincos(lib, shape):
    sin = torch.empty(shape.seq_len, shape.head_size, device="cuda")
    cos = torch.empty_like(sin)
    assert lib.kllm_sincos_init(shape.head_size, shape.seq_len, FLAVOURS[shape.flavour], ptr(sin), ptr(cos),
                                None) == 0
    sync()
    return sin, cos


def sequence(vocab, n, seed):
    toks = np.random.default_rng(seed).integers(0, vocab, n)
    toks[:3] = (1, 0, vocab - 1)
    return [int(t) for t in toks]


_CACHE = {}


def clear_cache():
    _CACHE.clear()
    torch.cuda.empty_cache()


def cached_model(lib, key, shape, weights, ends):
    """(shape, weights, tokens, plain model, fixed-point model or None) for `key`, the model's logits taken at
    `ends`; one geometry held at a time.  `weights` is a WEIGHTS name or a callable (device) -> weight dict."""
    if key not in _CACHE:
        clear_cache()
        w = WEIGHTS[weights](shape, "cuda", 77) if isinstance(weights, str) else weights("cuda")
        toks = sequence(shape.vocab_size, shape.seq_len, 5)
        sin, cos = device_sincos(lib, shape)
        plain = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends)
        fixed = None
        if shape.group_size == 64:
            fixed = prefill_ref(w, shape, toks, 0, sin, cos, tf32=False, logits_at=ends, fixed_point=True)
        _CACHE[key] = (shape, w, toks, plain, fixed)
    return _CACHE[key]


# ---- decoders and checks -------------------------------------------------------------------------------------------
def make_decoder(monkeypatch, shape, w, numerics, env, engine="persistent", kv_cache="fp32"):
    """A decoder with every engine knob cleared, then `env` set; `engine` None leaves the choice to the library.
    On the persistent engine, the attention geometry it reports must be engine_geometry's."""
    for name in KNOBS:
        monkeypatch.delenv(name, raising=False)
    if engine is not None:
        monkeypatch.setenv("KLLM_ENGINE", engine)
    for name, value in env.items():
        monkeypatch.setenv(name, value)
    dec = Decoder(shape, w, numerics=numerics, kv_cache=kv_cache)
    if engine is not None:
        assert dec.engine == engine
    if dec.engine == "persistent":
        want = engine_geometry(shape, numerics, env, sms(), kv_cache)
        assert dec.attention_geometry == want, (shape.name, numerics, env, kv_cache, dec.attention_geometry, want)
    return dec


def kv_ratios(got, ref, tau, tau_first):
    """Per-layer worst |got - ref| / (tau * rms(row)) over every position, for K and V; layer 0 against
    tau_first."""
    out = {}
    for name, g, r in (("K", got[0], ref["k"]), ("V", got[1], ref["v"])):
        g = torch.from_numpy(g).cuda().double()
        rms = r.pow(2).mean(-1, keepdim=True).sqrt()
        t = torch.full((r.shape[0], 1, 1), tau, dtype=torch.float64, device=r.device)
        t[0] = tau_first
        out[name] = [float(x) for x in ((g - r).abs() / (t * rms)).amax(dim=(1, 2))]
    return out


def logit_ratio(got, ref_logits, tau):
    return float((torch.from_numpy(got).cuda().double() - ref_logits).abs().max()) / (
        tau * float(ref_logits.pow(2).mean().sqrt()))


def fmt(per_layer):
    return {k: [float(f"{x:.3g}") for x in v] for k, v in per_layer.items()}


def run(what, dec, shape, toks, ref, ends, kv_tau, logit_tau, plain=None, kv_tau_first=KV_TAU_FIRST,
        tag="[decode-model]"):
    """Teacher-force toks over every position in segments ending at `ends`; check the logits at each end and
    every K / V row at the end.  Returns (the cache, {end: logits})."""
    start, worst_logit, worst_end, worst_plain = 0, 0.0, 0, 0.0
    logits = {}
    for end in ends:
        ids = dec.generate(0, start, end + 1 - start, teacher=toks[start:end + 1])
        got = dec.logits()
        logits[end] = got
        lref = ref["logits_at"][end]
        r = logit_ratio(got, lref, logit_tau)
        if r > worst_logit:
            worst_logit, worst_end = r, end
        top2 = torch.topk(lref, 2).values
        bound = logit_tau * float(lref.pow(2).mean().sqrt())
        if float(top2[0] - top2[1]) > 2 * bound:
            assert ids[-1] == int(torch.argmax(lref)), (what, end)
        if plain is not None:
            worst_plain = max(worst_plain, logit_ratio(got, plain["logits_at"][end], 1.0))
        start = end + 1
    assert start == shape.seq_len
    kv = dec.kv_cache()
    per_layer = kv_ratios(kv, ref, kv_tau, kv_tau_first)
    report(what, f"segments {ends}", tag=tag)
    report(what, f"logits err / bound {worst_logit:.3g}; K / V err / bound per layer {fmt(per_layer)}", tag=tag)
    if plain is not None:
        report(what, f"fixed point's cost, against the plain model: logits err / rms {worst_plain:.3g}; "
                     f"K / V err / rms per layer {fmt(kv_ratios(kv, plain, 1.0, 1.0))}", tag=tag)
    assert worst_logit <= 1.0, (what, worst_end, worst_logit)
    for name, v in per_layer.items():
        assert max(v) <= 1.0, (what, name, v)
    return kv, logits


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def compare_engines(what, shape, ends, a, b):
    """Two (cache, {end: logits}) results bit for bit; names the first differing layer and position."""
    (ka, la), (kb, lb) = a, b
    for end in ends:
        assert same_bits(la[end], lb[end]), (what, "logits", end)
    for name, x, y in (("K", ka[0], kb[0]), ("V", ka[1], kb[1])):
        for l in range(shape.layer_num):
            if not same_bits(x[l], y[l]):
                rows = np.nonzero((x[l].view(np.uint32) != y[l].view(np.uint32)).any(-1))[0]
                raise AssertionError(f"{what}: {name} layer {l} differs first at position {rows[0]}")
