"""ctypes front-end of the device-resident decoder (``kllm_decoder_*``) plus synthetic
random-init weights in the shapes BASELINE.json names.

torch is used here only as plumbing: device memory, RNG for the synthetic checkpoints and
stream handles.  All compute on the decode path happens inside libkllm_b200.so.
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass, replace

from . import DecoderDesc, FLAVOURS, KllmError, check, load_library
from .speculative import DEFAULT_DRAFT_LEN


@dataclass(frozen=True)
class ModelShape:
    """Header fields of a KuiperLLama checkpoint (kuiper/include/model/config.h:5-13)."""
    name: str
    dim: int
    hidden_dim: int
    layer_num: int
    head_num: int
    kv_head_num: int
    vocab_size: int
    seq_len: int
    shared_classifier: bool = False
    flavour: str = "llama2"
    group_size: int = 0  # 0 = fp32, 64 = export.py --version 3

    @property
    def head_size(self) -> int:
        return self.dim // self.head_num

    @property
    def kv_dim(self) -> int:
        return self.dim * self.kv_head_num // self.head_num

    @property
    def kv_mul(self) -> int:
        return self.head_num // self.kv_head_num

    def weight_bytes_per_token(self, weights: str = "fp32") -> int:
        """ALGORITHMIC bytes one decode step must read (SURVEY.md section 8d): every matmul
        weight once (+ int8 scales), the 2L+1 norm vectors, qkv biases and one embedding row.
        weights="bf16": the matrices of an fp32 checkpoint held in bf16 (Decoder(weight_format="bf16")), 2 bytes each."""
        d, h, L, kv, V = self.dim, self.hidden_dim, self.layer_num, self.kv_dim, self.vocab_size
        numel = L * (2 * d * d + 2 * kv * d + 3 * h * d) + V * d
        if weights not in ("fp32", "bf16") or (weights == "bf16" and self.group_size):
            raise ValueError(f"weights={weights!r} for {self.name}")
        if self.group_size:
            wbytes = numel + (numel // self.group_size) * 4
        else:
            wbytes = numel * (2 if weights == "bf16" else 4)
        extra = (2 * L + 1) * d * 4 + d * 4
        if self.flavour == "qwen2" and self.group_size == 0:
            extra += L * (d + 2 * kv) * 4
        return wbytes + extra

    def kv_bytes_at(self, pos: int, kv_cache: str = "fp32") -> int:
        """Bytes of the K and V rows 0 .. pos: 4 per element, 2 with kv_cache="bf16", 1 with "fp8"."""
        return 2 * self.layer_num * (pos + 1) * self.kv_dim * KV_ELEM_BYTES[kv_cache]


KV_ELEM_BYTES = {"fp32": 4, "bf16": 2, "fp8": 1}  # per cached element, by Decoder(kv_cache=...)


SHAPES = {
    # BASELINE.json configs (SURVEY.md section 8 table)
    "stories15m": ModelShape("stories15M-fp32", 288, 768, 6, 6, 6, 32000, 256, True),
    "tinyllama-1.1b": ModelShape("TinyLlama-1.1B-fp32", 2048, 5632, 22, 32, 4, 32000, 2048),
    "llama2-7b-int8": ModelShape("Llama-2-7B-int8-g64", 4096, 11008, 32, 32, 32, 32000, 2048,
                                 group_size=64),
    "qwen2.5-0.5b": ModelShape("Qwen2.5-0.5B-fp32", 896, 4864, 24, 14, 2, 151936, 32768, True,
                               flavour="qwen2"),
    "llama2-7b": ModelShape("Llama-2-7B-fp32", 4096, 11008, 32, 32, 32, 32000, 2048),
    # small shapes for parity tests
    "tiny": ModelShape("tiny-fp32", 64, 172, 2, 4, 2, 512, 64),
    "tiny-shared": ModelShape("tiny-shared-fp32", 64, 172, 2, 4, 4, 512, 64, True),
    "tiny-int8": ModelShape("tiny-int8", 128, 384, 2, 4, 2, 512, 64, group_size=64),
    "tiny-qwen": ModelShape("tiny-qwen2", 128, 344, 2, 4, 2, 640, 96, True, flavour="qwen2"),
    "small": ModelShape("small-fp32", 288, 768, 3, 9, 3, 4096, 160),
    "small-hs48": ModelShape("small-hs48-fp32", 288, 768, 3, 6, 6, 4096, 160),
    "small-int8": ModelShape("small-int8", 256, 768, 2, 4, 2, 1024, 96, group_size=64),
    "small-qwen": ModelShape("small-qwen2", 256, 704, 2, 4, 2, 1536, 128, True, flavour="qwen2"),
    # 8 heads / 2 kv heads: splits 2 ways (kv heads sharded) and 4 ways (kv heads replicated)
    "small-tp": ModelShape("small-tp-fp32", 256, 768, 3, 8, 2, 2048, 128),
    # int8 whose 2-way shards still give the persistent ring 16-byte scale rows
    "small-tp-int8": ModelShape("small-tp-int8", 512, 1536, 2, 8, 4, 1024, 96, group_size=64),
}


def quantize_q80(w, group_size: int):
    """tools/export.py:49-73 quantize_q80 on a torch tensor: symmetric int8 per group of
    `group_size` consecutive elements of the flattened tensor, scale = max|w|/127."""
    import torch
    flat = w.float().reshape(-1, group_size)
    wmax = flat.abs().max(dim=1).values
    scale = wmax / 127.0
    q = torch.round(flat / scale[:, None]).to(torch.int8)
    return q.reshape(w.shape), scale.contiguous()


def synth_weights(shape: ModelShape, device="cuda", seed: int = 1234, norm_jitter: float = 0.1):
    """Random-init weights following tools/model.py:233-247 (N(0,0.02^2); wo and w3 scaled by
    1/sqrt(2L)), generated on `device`.  Norm weights are 1 + U(-j, j) so the norm multiply is
    actually exercised.  Returns a dict of contiguous torch tensors (int8 + scales if quant)."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    s = shape
    L, d, h, kv, V = s.layer_num, s.dim, s.hidden_dim, s.kv_dim, s.vocab_size

    def normal(*dims, std=0.02):
        return torch.empty(*dims, device=device, dtype=torch.float32).normal_(0.0, std, generator=g)

    def norm_w(*dims):
        w = torch.ones(*dims, device=device, dtype=torch.float32)
        if norm_jitter:
            w += (torch.rand(*dims, device=device, generator=g) * 2 - 1) * norm_jitter
        return w

    small = 0.02 / math.sqrt(2 * L)
    w = {
        "tok_emb": normal(V, d),
        "attn_norm": norm_w(L, d), "ffn_norm": norm_w(L, d), "final_norm": norm_w(d),
        "wq": normal(L, d, d), "wk": normal(L, kv, d), "wv": normal(L, kv, d),
        "wo": normal(L, d, d, std=small),
        "w1": normal(L, h, d), "w2": normal(L, d, h), "w3": normal(L, h, d, std=small),
    }
    w["wcls"] = None if s.shared_classifier else normal(V, d)
    if s.flavour == "qwen2" and s.group_size == 0:
        w["bq"], w["bk"], w["bv"] = normal(L, d), normal(L, kv), normal(L, kv)
    if s.group_size:
        if s.shared_classifier:
            raise KllmError("int8 + shared classifier is a reference defect (llama3.cpp:259-277)")
        for name in ("wq", "wk", "wv", "wo", "w1", "w2", "w3", "wcls"):
            qs = [quantize_q80(t, s.group_size) for t in (w[name] if name != "wcls" else [w[name]])]
            q = torch.stack([a for a, _ in qs])
            sc = torch.stack([b for _, b in qs])
            if name == "wcls":
                q, sc = q[0], sc[0]
            w[name], w["s" + name[1:]] = q.contiguous(), sc.contiguous()
    return w


MATRICES = ("wq", "wk", "wv", "wo", "w1", "w2", "w3")


def bf16_weights(weights: dict) -> dict:
    """The weight dict Decoder(weight_format="bf16") takes, from an fp32 one (synth_weights or a checkpoint's): the matrices
    and the classifier rounded to bf16, round to nearest even (torch's conversion); with a shared classifier
    ("wcls" None) a separate bf16 copy of the embedding.  tok_emb, the norms and the Qwen2 biases stay fp32."""
    import torch
    if "sq" in weights:
        raise KllmError("bf16 weights are for fp32 checkpoints, not int8 ones")
    out = dict(weights)
    for n in MATRICES:
        out[n] = weights[n].to(torch.bfloat16).contiguous()
    wcls = weights.get("wcls")
    out["wcls"] = (wcls if wcls is not None else weights["tok_emb"]).to(torch.bfloat16).contiguous()
    return out


def widen_weights(weights16: dict) -> dict:
    """bf16_weights' result widened back to fp32 (exact): the fp32 decoder over these weights is what a bf16-weight
    decoder reproduces bit for bit.  The classifier is always given explicitly (never None)."""
    import torch
    out = dict(weights16)
    for n in MATRICES + ("wcls",):
        out[n] = weights16[n].to(torch.float32).contiguous()
    return out


FP8_MAX = 448.0  # the largest finite e4m3 value


def fp8_kv_scales(k, v, kv_heads=None):
    """Calibrated scales for Decoder(kv_cache="fp8", kv_scales=...): amax / 448 per (layer, KV head) of the (key,
    value) arrays Decoder.kv_cache() returns from an fp32-cache run, so that the largest element of each maps to
    the largest finite e4m3 value; 1 where the amax is 0.  k and v are [L, seq_len, kv_dim] with `kv_heads` heads
    (or already [L, seq_len, kv_heads, head_size]).  Returns float32 numpy [2, L, kv_heads]: the K scales, then the
    V scales."""
    import numpy as np
    out = []
    for a in (k, v):
        a = np.asarray(a, dtype=np.float32)
        if a.ndim == 3:
            if kv_heads is None or a.shape[2] % kv_heads:
                raise ValueError(f"kv_heads={kv_heads!r} for arrays of shape {a.shape}")
            a = a.reshape(a.shape[0], a.shape[1], kv_heads, a.shape[2] // kv_heads)
        amax = np.abs(a).max(axis=(1, 3))
        out.append(np.where(amax > 0, amax / np.float32(FP8_MAX), np.float32(1.0)).astype(np.float32))
    return np.stack(out)


def _ptr_array(tensors):
    arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    return arr


def _relay(on_tokens, callback_type):
    """The `callback_type` callback that hands each call's ids to on_tokens (its leading arguments, then the ids as a
    list), or a null one for on_tokens None; and the list that keeps what on_tokens raised.  An exception cannot cross
    the C frames: the caller re-raises errors[0] after the call."""
    errors = []
    if on_tokens is None:
        return callback_type(), errors

    def relay(_ctx, *args):
        *lead, ids, n = args
        try:
            on_tokens(*lead, [ids[i] for i in range(n)])
        except BaseException as e:
            errors.append(e)

    return callback_type(relay), errors


class Decoder:
    """Owns a ``kllm_decoder`` built over torch-held device weights."""

    def __init__(self, shape: ModelShape, weights: dict, stream=None, tp_size=1, tp_rank=0,
                 allreduce=None, allreduce_ctx=None, full_dim=None, comm=None, numerics="exact",
                 kv_cache="fp32", weight_format="fp32", kv_scales=None):
        self.lib = load_library()
        self.shape = shape
        self.weights = weights  # keep the tensors alive
        s = shape
        L = s.layer_num
        d = DecoderDesc()
        d.dim = full_dim or s.dim
        d.hidden_dim, d.layer_num = s.hidden_dim, L
        d.head_num, d.kv_head_num = s.head_num, s.kv_head_num
        d.vocab_size, d.seq_len = s.vocab_size, s.seq_len
        d.flavour = FLAVOURS[s.flavour]
        d.group_size = s.group_size
        self._keep = []

        def per_layer(t):
            arr = _ptr_array([t[l] for l in range(L)])
            self._keep.append(arr)
            return ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p))

        d.tok_emb = weights["tok_emb"].data_ptr()
        d.attn_norm, d.ffn_norm = per_layer(weights["attn_norm"]), per_layer(weights["ffn_norm"])
        d.final_norm = weights["final_norm"].data_ptr()
        for n in ("wq", "wk", "wv", "wo", "w1", "w2", "w3"):
            setattr(d, n, per_layer(weights[n]))
        wcls = weights.get("wcls")
        d.wcls = (wcls if wcls is not None else weights["tok_emb"]).data_ptr()
        if s.group_size:
            for n in ("sq", "sk", "sv", "so", "s1", "s2", "s3"):
                setattr(d, n, per_layer(weights[n]))
            d.scls = weights["scls"].data_ptr()
        if "bq" in weights:
            d.bq, d.bk, d.bv = (per_layer(weights[n]) for n in ("bq", "bk", "bv"))
        d.tp_size, d.tp_rank = tp_size, tp_rank
        # "exact": bit-identical to the reference; "fast": toleranced (kllm_b200.h, kllm_decoder_desc::numerics)
        d.numerics = {"exact": 0, "fast": 1}[numerics]
        # "fp32": the cache of every other mode; "bf16": rows rounded to bf16 as they are cached; "fp8": rows stored as
        # e4m3 codes at a scale per (layer, KV head), kv_scales [2, L, kv_heads] (None: all 1; fp8_kv_scales
        # calibrates them).  Both fast numerics on the persistent engine only (kllm_b200.h, kllm_decoder_desc::kv_cache)
        d.kv_cache = {"fp32": 0, "bf16": 1, "fp8": 2}[kv_cache]
        if kv_cache == "fp8" and kv_scales is None:
            import numpy as np
            kv_scales = np.ones((2, L, s.kv_head_num), np.float32)  # the C ABI takes unit scales as an array of ones
        if kv_scales is not None:
            import numpy as np
            sc = np.ascontiguousarray(np.asarray(kv_scales, dtype=np.float32))
            if sc.shape != (2, L, s.kv_head_num):
                raise KllmError(f"kv_scales of shape {sc.shape}, not (2, {L}, {s.kv_head_num})")
            self._kv_scales = sc  # read by kllm_decoder_create only
            d.kv_scales = sc.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
        # "bf16": the matrices and wcls are bf16 tensors (bf16_weights), the arithmetic fp32 (kllm_decoder_desc::weights)
        d.weights = {"fp32": 0, "bf16": 1}[weight_format]
        want = "torch.bfloat16" if weight_format == "bf16" else None
        for n in MATRICES + ("wcls",):
            t = weights.get(n)
            if t is not None and (str(t.dtype) == "torch.bfloat16") != (want is not None):
                raise KllmError(f"weight_format={weight_format!r} with {n} of {t.dtype} (decoder.bf16_weights)")
        if weight_format == "bf16" and weights.get("wcls") is None:
            raise KllmError("weight_format='bf16' needs its own bf16 wcls (decoder.bf16_weights)")
        if allreduce is not None:
            d.allreduce = allreduce
            d.allreduce_ctx = allreduce_ctx
        if comm is not None:
            d.comm = comm.handle
            self.comm = comm  # keep alive
        self.desc = d
        self._top_n = -1  # kllm_decoder_set_logprobs's setting (a new decoder's is off)
        # local head geometry (head counts in `shape` are per-rank under tensor parallelism)
        self.head_size = d.dim // (s.head_num * max(tp_size, 1))
        self.local_kv_dim = s.kv_head_num * self.head_size
        handle = ctypes.c_void_p()
        stream_ptr = ctypes.c_void_p(stream) if stream else None
        check(self.lib.kllm_decoder_create(ctypes.byref(d), stream_ptr, ctypes.byref(handle)),
              "kllm_decoder_create")
        self.handle = handle

    def close(self):
        if getattr(self, "handle", None):
            self.lib.kllm_decoder_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches_per_step(self) -> int:
        return self.lib.kllm_decoder_launches_per_step(self.handle)

    @property
    def classifier_rows(self) -> int:
        """Classifier rows this rank streams per token (vocab / tp when sharded by vocabulary)."""
        return self.lib.kllm_decoder_classifier_rows(self.handle)

    @property
    def engine(self) -> str:
        return self.lib.kllm_decoder_engine(self.handle).decode()

    @property
    def attention_geometry(self):
        """(tile, split, tile_v, stage_bytes) of the persistent engine's attention
        (kllm_decoder_attention_geometry); KllmError on the graph engine."""
        out = [ctypes.c_int(0) for _ in range(4)]
        check(self.lib.kllm_decoder_attention_geometry(self.handle, *[ctypes.byref(v) for v in out]),
              "kllm_decoder_attention_geometry")
        return tuple(v.value for v in out)

    def step(self, token: int, pos: int, is_prompt: bool = False) -> int:
        """Reference-facing call with host buffers (predict + post_processing)."""
        nxt = ctypes.c_int32(-1)
        check(self.lib.kllm_decoder_step(self.handle, token, pos, int(is_prompt), ctypes.byref(nxt)),
              "kllm_decoder_step")
        return nxt.value

    def _feed(self, entry: str, tokens, start_pos: int) -> int:
        """Calls the prompt-style C entry `entry` (tokens, n, start_pos, &next) and returns next."""
        n = len(tokens)
        arr = (ctypes.c_int32 * n)(*[int(t) for t in tokens])
        nxt = ctypes.c_int32(-1)
        check(getattr(self.lib, entry)(self.handle, arr, n, start_pos, ctypes.byref(nxt)), entry)
        return nxt.value

    def prompt(self, tokens, start_pos: int = 0) -> int:
        """Feed a whole prompt (one launch on the persistent engine, classifier only for the last
        position); returns the greedy id that follows the prompt."""
        return self._feed("kllm_decoder_prompt", tokens, start_pos)

    def prefill_tf32(self, tokens, start_pos: int = 0) -> int:
        """TOLERANCED batched prefill on the Hopper tensor cores (wgmma) (TF32); same contract as prompt()."""
        return self._feed("kllm_decoder_prefill_tf32", tokens, start_pos)

    def prefill_w8(self, tokens, start_pos: int = 0) -> int:
        """TOLERANCED batched prefill of an int8 checkpoint: the weight tiles are dequantised to TF32 on the way
        to the same wgmma GEMM as prefill_tf32(); same contract as prompt()."""
        return self._feed("kllm_decoder_prefill_w8", tokens, start_pos)

    def generate(self, first_token: int, start_pos: int, n_steps: int, teacher=None):
        out = (ctypes.c_int32 * n_steps)()
        tf = None
        if teacher is not None:
            tf = (ctypes.c_int32 * n_steps)(*[int(t) for t in teacher[:n_steps]])
        check(self.lib.kllm_decoder_generate(self.handle, first_token, start_pos, n_steps, tf, out),
              "kllm_decoder_generate")
        return list(out)

    def generate_until(self, first_token: int, start_pos: int, max_steps: int, stop_ids=(), on_tokens=None):
        """Generate from `first_token` at `start_pos` until the first id in `stop_ids` (included in the result) or
        `max_steps` ids (kllm_decoder_generate_until).  `on_tokens(list_of_ints)` receives every id exactly once,
        in order, while the loop runs; it must not call into this decoder."""
        from . import TOKEN_CALLBACK
        stops = [int(t) for t in stop_ids]
        sarr = (ctypes.c_int32 * max(len(stops), 1))(*stops)
        out = (ctypes.c_int32 * max(int(max_steps), 1))()
        n_out = ctypes.c_int32(0)
        cb, errors = _relay(on_tokens, TOKEN_CALLBACK)
        check(self.lib.kllm_decoder_generate_until(self.handle, int(first_token), int(start_pos), int(max_steps),
                                                   sarr, len(stops), cb, None, out, ctypes.byref(n_out)),
              "kllm_decoder_generate_until")
        if errors:
            raise errors[0]
        return list(out[:n_out.value])

    def verify(self, tokens, start_pos: int):
        """Speculative decoding's verify pass (kllm_decoder_verify): tokens[0] fed at start_pos, tokens[1:] drafts for
        the positions after it, all in one pass over the weights.  Returns id_0 .. id_a, the ids drawn at
        start_pos .. start_pos + a, where a is the number of leading drafts equal to the id drawn before them: bit for
        bit generate(tokens[0], start_pos, a + 1)."""
        toks = [int(t) for t in tokens]
        arr = (ctypes.c_int32 * max(len(toks), 1))(*toks)
        out = (ctypes.c_int32 * max(len(toks), 1))()
        a = ctypes.c_int32(0)
        check(self.lib.kllm_decoder_verify(self.handle, arr, len(toks), int(start_pos), out, ctypes.byref(a)),
              "kllm_decoder_verify")
        return list(out[:a.value + 1])

    def generate_speculative(self, first_token: int, start_pos: int, max_steps: int, stop_ids=(), on_tokens=None,
                             draft_len: int = DEFAULT_DRAFT_LEN, ngram_max: int = 3):
        """generate_until with prompt-lookup drafts checked by verify passes (kllm_decoder_generate_speculative):
        the same ids, logits, history, record and cache rows.  Returns (ids, stats) with stats a dict of rounds,
        drafted and accepted (speculative.simulate_rounds predicts them)."""
        from . import TOKEN_CALLBACK, SpecStats
        stops = [int(t) for t in stop_ids]
        sarr = (ctypes.c_int32 * max(len(stops), 1))(*stops)
        out = (ctypes.c_int32 * max(int(max_steps), 1))()
        n_out = ctypes.c_int32(0)
        stats = SpecStats()
        cb, errors = _relay(on_tokens, TOKEN_CALLBACK)
        check(self.lib.kllm_decoder_generate_speculative(self.handle, int(first_token), int(start_pos), int(max_steps),
                                                         sarr, len(stops), int(draft_len), int(ngram_max), cb, None,
                                                         out, ctypes.byref(n_out), ctypes.byref(stats)),
              "kllm_decoder_generate_speculative")
        if errors:
            raise errors[0]
        return list(out[:n_out.value]), {"rounds": stats.rounds, "drafted": stats.drafted,
                                         "accepted": stats.accepted}

    def copy_prefix(self, src: "Decoder", n_pos: int):
        """Copy src's K/V rows, history and record entries of positions [0, n_pos) into this decoder
        (kllm_decoder_copy_prefix): an entry here that continues at a position <= n_pos then returns what it would on
        src, under this decoder's own draw settings.  Both must describe the same model on the same engine and
        cache."""
        check(self.lib.kllm_decoder_copy_prefix(self.handle, src.handle, int(n_pos)), "kllm_decoder_copy_prefix")

    def set_sampling(self, temperature: float, top_k: int = 0, seed: int = 0, top_p: float = 1.0):
        """Draw every later id by the sampling rule (kllm_decoder_set_sampling; sampling.py mirrors it)
        instead of the greedy argmax; temperature 0 is greedy again.  top_p < 1 adds nucleus sampling after
        top-k (kllm_decoder_set_sampling_top_p)."""
        if top_p == 1.0:
            check(self.lib.kllm_decoder_set_sampling(self.handle, float(temperature), int(top_k), int(seed)),
                  "kllm_decoder_set_sampling")
        else:
            check(self.lib.kllm_decoder_set_sampling_top_p(self.handle, float(temperature), int(top_k),
                                                           float(top_p), int(seed)),
                  "kllm_decoder_set_sampling_top_p")

    def set_repetition_penalty(self, penalty: float, last_n: int = 0):
        """Penalise, before every later draw, the logits of the ids fed at the last `last_n` positions (0: the whole
        sequence), as HF's RepetitionPenaltyLogitsProcessor does (kllm_decoder_set_repetition_penalty;
        sampling.penalize mirrors it).  penalty 1 is off; the sampling settings are left alone."""
        check(self.lib.kllm_decoder_set_repetition_penalty(self.handle, float(penalty), int(last_n)),
              "kllm_decoder_set_repetition_penalty")

    def set_frequency_presence(self, frequency: float, presence: float, from_pos: int = 0):
        """Subtract, before every later draw, frequency * c_i and then presence from the logit of every id fed
        c_i > 0 times at positions [from_pos, pos] (OpenAI's frequency_penalty / presence_penalty; from_pos = the
        prompt's length counts the generated ids only).  0, 0 is off; the other settings are left alone
        (kllm_decoder_set_frequency_presence; sampling.frequency_presence mirrors it)."""
        check(self.lib.kllm_decoder_set_frequency_presence(self.handle, float(frequency), float(presence),
                                                           int(from_pos)), "kllm_decoder_set_frequency_presence")

    def set_logit_bias(self, mapping=None):
        """Add mapping[id] to the logit of each id before every later draw (OpenAI's logit_bias), replacing the
        map in force; None or {} clears it (kllm_decoder_set_logit_bias; sampling.apply_bias mirrors it)."""
        mapping = mapping or {}
        ids = (ctypes.c_int32 * max(1, len(mapping)))(*[int(i) for i in mapping])
        vals = (ctypes.c_float * max(1, len(mapping)))(*[float(b) for b in mapping.values()])
        check(self.lib.kllm_decoder_set_logit_bias(self.handle, ids, vals, len(mapping)),
              "kllm_decoder_set_logit_bias")

    def set_logprobs(self, top_n: int):
        """Record, at every position whose classifier runs, the returned id's log-probability over the raw logits and,
        for top_n > 0, the top_n alternatives (kllm_decoder_set_logprobs; sampling.logprobs mirrors the rule).  -1 is
        off.  Clears the record."""
        check(self.lib.kllm_decoder_set_logprobs(self.handle, int(top_n)), "kllm_decoder_set_logprobs")
        self._top_n = int(top_n)

    def logprobs(self, start_pos: int, n: int):
        """The record of positions [start_pos, start_pos + n) (kllm_decoder_read_logprobs): numpy (ids [n], lp [n],
        top_ids [n, top_n], top_lp [n, top_n]); an id of -1 marks a position without an entry."""
        import numpy as np
        k = max(self._top_n, 0)
        ids = np.empty(n, np.int32)
        lp = np.empty(n, np.float32)
        top_ids = np.empty((n, k), np.int32)
        top_lp = np.empty((n, k), np.float32)
        vp = ctypes.c_void_p
        check(self.lib.kllm_decoder_read_logprobs(self.handle, int(start_pos), int(n), ids.ctypes.data_as(vp),
                                                  lp.ctypes.data_as(vp), top_ids.ctypes.data_as(vp) if k else None,
                                                  top_lp.ctypes.data_as(vp) if k else None),
              "kllm_decoder_read_logprobs")
        return ids, lp, top_ids, top_lp

    def score(self, tokens, start_pos: int = 0):
        """Teacher-forced log-likelihood (kllm_decoder_score): lp[i] = log p(tokens[i + 1] | tokens[:i + 1]) with
        tokens[0] at start_pos, n - 1 values as numpy fp32.  The cache then holds those positions."""
        import numpy as np
        n = len(tokens)
        arr = (ctypes.c_int32 * max(n, 1))(*[int(t) for t in tokens])
        lp = np.empty(max(n - 1, 1), np.float32)
        check(self.lib.kllm_decoder_score(self.handle, arr, n, int(start_pos), lp.ctypes.data_as(ctypes.c_void_p)),
              "kllm_decoder_score")
        return lp[:n - 1]

    def history(self):
        """The id fed at each position [seq_len], -1 where none was (kllm_decoder_read_history)."""
        import numpy as np
        buf = np.empty(self.shape.seq_len, dtype=np.int32)
        check(self.lib.kllm_decoder_read_history(self.handle, buf.ctypes.data_as(ctypes.c_void_p)),
              "kllm_decoder_read_history")
        return buf

    def logits(self):
        import numpy as np
        buf = np.empty(self.shape.vocab_size, dtype=np.float32)
        check(self.lib.kllm_decoder_logits(self.handle, buf.ctypes.data_as(ctypes.c_void_p)),
              "kllm_decoder_logits")
        return buf

    def kv_cache(self):
        """(key, value) caches as numpy arrays [L, seq_len, kv_dim] in the reference layout."""
        import numpy as np
        s = self.shape
        k = np.empty((s.layer_num, s.seq_len, self.local_kv_dim), np.float32)
        v = np.empty_like(k)
        check(self.lib.kllm_decoder_read_kv(self.handle, k.ctypes.data_as(ctypes.c_void_p),
                                            v.ctypes.data_as(ctypes.c_void_p)), "kllm_decoder_read_kv")
        return k, v


class Batch:
    """Owns a ``kllm_batch``: up to MAX_BATCH decoders over one model, stepped in one pass over the weights per step.
    Each member ends bit for bit as its own step / generate with the same arguments would leave it (kllm_b200.h).
    Close the batch before its members."""

    def __init__(self, decoders, stream=None):
        self.lib = load_library()
        self.members = list(decoders)  # keep the decoders alive while the batch is
        n = len(self.members)
        arr = (ctypes.c_void_p * max(n, 1))(*[d.handle.value if d.handle else None for d in self.members])
        handle = ctypes.c_void_p()
        stream_ptr = ctypes.c_void_p(stream) if stream else None
        check(self.lib.kllm_batch_create(arr, n, stream_ptr, ctypes.byref(handle)), "kllm_batch_create")
        self.handle = handle

    def _rows(self, values):
        vals = [int(v) for v in values]
        if len(vals) != len(self.members):
            raise KllmError(f"{len(vals)} values for {len(self.members)} members")
        return (ctypes.c_int32 * len(vals))(*vals)

    def step(self, tokens, positions):
        """One step of every member: tokens[b] fed at positions[b]; returns member b's id at b."""
        out = (ctypes.c_int32 * len(self.members))()
        check(self.lib.kllm_batch_step(self.handle, self._rows(tokens), self._rows(positions), out),
              "kllm_batch_step")
        return list(out)

    def generate(self, first_tokens, start_positions, n_steps: int):
        """n_steps steps of every member (kllm_batch_generate); returns one list of n_steps ids per member."""
        n = len(self.members)
        out = (ctypes.c_int32 * (n * max(int(n_steps), 1)))()
        check(self.lib.kllm_batch_generate(self.handle, self._rows(first_tokens), self._rows(start_positions),
                                           int(n_steps), out), "kllm_batch_generate")
        return [list(out[b * n_steps:(b + 1) * n_steps]) for b in range(n)]

    def generate_until(self, first_tokens, start_positions, max_steps, stop_ids, on_tokens=None):
        """Member b generates from first_tokens[b] at start_positions[b] until the first id in stop_ids[b] (included)
        or max_steps[b] ids, and ends as its own Decoder.generate_until would leave it; each pass carries only the
        members still running (kllm_batch_generate_until).  `on_tokens(member, list_of_ints)` receives every id of
        every member exactly once, in order per member, while the loop runs; it must not call into the batch or its
        members.  Returns (one list of ids per member, {"passes": .., "rows": ..})."""
        from . import BATCH_TOKEN_CALLBACK, MAX_STOP_IDS, BatchStats
        n = len(self.members)
        steps = self._rows(max_steps)
        if len(stop_ids) != n:
            raise KllmError(f"{len(stop_ids)} stop lists for {n} members")
        stops = (ctypes.c_int32 * (n * MAX_STOP_IDS))()
        n_stop = (ctypes.c_int32 * n)()
        for b, ids in enumerate(stop_ids):
            ids = [int(t) for t in ids]
            if len(ids) > MAX_STOP_IDS:
                raise KllmError(f"member {b}: {len(ids)} stop ids, at most {MAX_STOP_IDS}")
            stops[b * MAX_STOP_IDS:b * MAX_STOP_IDS + len(ids)] = ids
            n_stop[b] = len(ids)
        M = max(list(steps) + [1])
        out = (ctypes.c_int32 * (n * M))()
        n_out = (ctypes.c_int32 * n)()
        stats = BatchStats()
        cb, errors = _relay(on_tokens, BATCH_TOKEN_CALLBACK)
        check(self.lib.kllm_batch_generate_until(self.handle, self._rows(first_tokens), self._rows(start_positions),
                                                 steps, stops, n_stop, cb, None, out, n_out, ctypes.byref(stats)),
              "kllm_batch_generate_until")
        if errors:
            raise errors[0]
        return ([list(out[b * M:b * M + n_out[b]]) for b in range(n)],
                {"passes": stats.passes, "rows": stats.rows})

    def beam_search(self, first_token: int, start_pos: int, max_new_tokens: int, eos_ids=(),
                    length_penalty: float = 1.0, early_stopping=False, n_return: int = 1):
        """Beam search with one beam per member (kllm_batch_beam_search): transformers' generate(num_beams=B,
        length_penalty, early_stopping, num_return_sequences=n_return) with no logits processors, the rule of
        beam.py.  Member 0 holds the prompt's positions [0, start_pos); first_token is fed at start_pos.
        early_stopping is False, True or "never"; length_penalty is passed as fp32.  Returns ([{"ids", "score",
        "sum"}, ...] best first, {"passes", "forks", "fork_rows"})."""
        from . import BeamStats
        from .beam import early_stopping_code
        eos = [int(t) for t in eos_ids]
        earr = (ctypes.c_int32 * max(len(eos), 1))(*eos)
        steps, n_ret = max(int(max_new_tokens), 1), max(int(n_return), 1)
        out = (ctypes.c_int32 * (n_ret * steps))()
        lens = (ctypes.c_int32 * n_ret)()
        scores = (ctypes.c_float * n_ret)()
        sums = (ctypes.c_float * n_ret)()
        stats = BeamStats()
        check(self.lib.kllm_batch_beam_search(self.handle, int(first_token), int(start_pos), int(max_new_tokens),
                                              earr, len(eos), float(length_penalty),
                                              early_stopping_code(early_stopping), int(n_return), out, lens, scores,
                                              sums, ctypes.byref(stats)), "kllm_batch_beam_search")
        hyps = [{"ids": list(out[i * steps:i * steps + lens[i]]), "score": scores[i], "sum": sums[i]}
                for i in range(int(n_return))]
        return hyps, {"passes": stats.passes, "forks": stats.forks, "fork_rows": stats.fork_rows}

    def close(self):
        if getattr(self, "handle", None):
            self.lib.kllm_batch_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
