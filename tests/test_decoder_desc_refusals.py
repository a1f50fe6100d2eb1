"""kllm_decoder_create's refusals of a bad model description, without a GPU.  Every description check comes before
the decoder looks for a device, so each refusal returns its code on any machine; a description that breaks two
rules returns the code of the first check it fails (kllm_b200.h keeps that order part of the interface)."""
import ctypes

import pytest

from kuiperllama_b200 import DecoderDesc

E_INVALID, E_UNSUPPORTED, E_NODEVICE = -1, -2, -4
L = 2
MATRICES = ("wq", "wk", "wv", "wo", "w1", "w2", "w3")
SCALES = ("sq", "sk", "sv", "so", "s1", "s2", "s3")

_keep = []


def _per_layer(base):
    arr = (ctypes.c_void_p * L)(*[base + 0x10000 * l for l in range(L)])
    _keep.append(arr)
    return ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p))


def valid_desc(group_size=0, qwen2=False):
    """A description no check refuses.  The pointers are never dereferenced: every refusal comes first."""
    d = DecoderDesc()
    d.dim, d.hidden_dim, d.layer_num, d.head_num, d.kv_head_num = 64, 128, L, 4, 2
    d.vocab_size, d.seq_len, d.flavour, d.group_size = 32, 16, 0, group_size
    d.tok_emb, d.final_norm, d.wcls = 0x100000, 0x200000, 0x300000
    d.attn_norm, d.ffn_norm = _per_layer(0x400000), _per_layer(0x500000)
    for i, n in enumerate(MATRICES):
        setattr(d, n, _per_layer(0x1000000 * (i + 1)))
    if group_size:
        for i, n in enumerate(SCALES):
            setattr(d, n, _per_layer(0x10000000 + 0x1000000 * i))
        d.scls = 0x600000
    if qwen2:
        d.bq, d.bk, d.bv = _per_layer(0x700000), _per_layer(0x800000), _per_layer(0x900000)
    d.tp_size, d.tp_rank = 1, 0
    return d


def create(lib, d):
    handle = ctypes.c_void_p()
    return lib.kllm_decoder_create(ctypes.byref(d), None, ctypes.byref(handle))


def _set(**fields):
    return lambda d: [setattr(d, k, v) for k, v in fields.items()]


def _null(name):
    return lambda d: setattr(d, name, None)


def _tp(size):
    # a second rank with its all-reduce callback, so that only the rule under test refuses
    def apply(d):
        d.tp_size, d.tp_rank, d.allreduce_ctx = size, 0, None
        d.comm = 0x1234
    return apply


CASES = {
    # sizes
    "zero_dim": (0, _set(dim=0), E_INVALID),
    "negative_seq_len": (0, _set(seq_len=-1), E_INVALID),
    # null pointers
    "null_tok_emb": (0, _null("tok_emb"), E_INVALID),
    "null_attn_norm": (0, _null("attn_norm"), E_INVALID),
    "null_ffn_norm": (0, _null("ffn_norm"), E_INVALID),
    "null_final_norm": (0, _null("final_norm"), E_INVALID),
    "null_wcls": (0, _null("wcls"), E_INVALID),
    **{f"null_{n}": (0, _null(n), E_INVALID) for n in MATRICES},
    # int8 without its scales
    **{f"int8_null_{n}": (64, _null(n), E_INVALID) for n in SCALES + ("scls",)},
    # shape
    "head_num_not_dividing_dim": (0, _set(head_num=3, kv_head_num=1), E_INVALID),
    "kv_heads_not_dividing_heads": (0, _set(kv_head_num=3), E_INVALID),
    "dim_not_multiple_of_4": (0, _set(dim=66, head_num=2, kv_head_num=1), E_UNSUPPORTED),
    "hidden_not_multiple_of_4": (0, _set(hidden_dim=130), E_UNSUPPORTED),
    # storage formats
    "kv_cache_out_of_range": (0, _set(kv_cache=2), E_INVALID),
    "kv_cache_negative": (0, _set(kv_cache=-1), E_INVALID),
    "weights_out_of_range": (0, _set(weights=2), E_INVALID),
    "weights_negative": (0, _set(weights=-1), E_INVALID),
    "bf16_weights_with_int8": (64, _set(weights=1), E_INVALID),
    # tensor parallel
    "tp_without_transport": (0, _set(tp_size=2), E_INVALID),
    "tp_head_num_not_dividing_dim": (0, lambda d: (_tp(2)(d), _set(head_num=64, kv_head_num=64)(d)), E_INVALID),
    "bf16_weights_tp": (0, lambda d: (_tp(2)(d), _set(weights=1)(d)), E_UNSUPPORTED),
    "bf16_cache_tp": (0, lambda d: (_tp(2)(d), _set(kv_cache=1)(d)), E_UNSUPPORTED),
    # two rules at once: the first check decides
    "null_wq_and_dim_not_multiple_of_4": (0, lambda d: (_null("wq")(d), _set(dim=66, head_num=2, kv_head_num=1)(d)),
                                          E_INVALID),
    "bf16_weights_with_int8_and_tp": (64, lambda d: (_tp(2)(d), _set(weights=1)(d)), E_INVALID),
    "dim_not_multiple_of_4_and_weights_out_of_range": (0, _set(dim=66, head_num=2, kv_head_num=1, weights=5),
                                                       E_UNSUPPORTED),
    "kv_cache_and_weights_out_of_range": (0, _set(kv_cache=7, weights=7), E_INVALID),
    "kv_cache_out_of_range_and_bf16_weights_tp": (0, lambda d: (_tp(2)(d), _set(weights=1, kv_cache=3)(d)), E_INVALID),
    "bf16_weights_and_bf16_cache_tp": (0, lambda d: (_tp(2)(d), _set(weights=1, kv_cache=1)(d)), E_UNSUPPORTED),
    "int8_null_scale_and_bf16_weights": (64, lambda d: (_null("s2")(d), _set(weights=1)(d)), E_INVALID),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_bad_description_is_refused(kllm_lib, case):
    group_size, edit, code = CASES[case]
    d = valid_desc(group_size)
    edit(d)
    assert create(kllm_lib, d) == code


def test_bf16_cache_on_the_graph_engine_is_refused(kllm_lib, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", "graph")
    d = valid_desc()
    d.kv_cache = 1
    assert create(kllm_lib, d) == E_UNSUPPORTED


def _device_visible():
    try:
        import torch
        return torch.cuda.device_count() > 0
    except Exception:
        return False


@pytest.mark.parametrize("group_size,qwen2,weights,kv_cache", [(0, False, 0, 0), (64, False, 0, 0), (0, True, 0, 0),
                                                                (0, False, 1, 0), (0, False, 0, 1), (0, False, 1, 1)])
def test_valid_description_reaches_the_device_lookup(kllm_lib, group_size, qwen2, weights, kv_cache):
    if _device_visible():
        pytest.skip("a device is present: the description's fake pointers must not reach it")
    d = valid_desc(group_size, qwen2)
    d.weights, d.kv_cache = weights, kv_cache
    assert create(kllm_lib, d) == E_NODEVICE
