"""The persistent engine's kernel table: every decode_megakernel<F, KV, LP, PROF> instantiation the library holds
(megakernel.cu, kernels_for).  tests/test_abi.py checks each one's SASS; tests/test_megakernel_coverage.py checks that
each non-profiling one runs in at least one GPU case held to the fp64 model or to the log-probability mirror.

Entries are (weight format, KV cache, log-probabilities, profiling): {fp32, int8, bf16} weights x {fp32, bf16, fp8}
caches x {plain, log-probabilities}, plus the profiling kernels of fp32 and int8 weights over the fp32 cache.
"""
WEIGHT_FORMATS = ("fp32", "int8", "bf16")  # WeightFormat (decoder_model.h), in enum order
KV_CACHES = ("fp32", "bf16", "fp8")  # kllm_decoder_desc::kv_cache, in enum order

TABLE = [(f, kv, lp, False) for f in WEIGHT_FORMATS for kv in KV_CACHES for lp in (False, True)] + \
        [(f, "fp32", False, True) for f in ("fp32", "int8")]
MODEL_CHECKED = [(f, kv, lp) for f, kv, lp, prof in TABLE if not prof]


def symbol(f, kv, lp, prof):
    """The mangled name of kllm::mega::decode_megakernel<F, KV, LP, PROF>(Params)."""
    return "_ZN4kllm4mega17decode_megakernelILNS_12WeightFormatE{}ELi{}ELb{}ELb{}EEEvNS0_6ParamsE".format(
        WEIGHT_FORMATS.index(f), KV_CACHES.index(kv), int(lp), int(prof))


def row(f, kv, lp):
    """A table row as people read it, for failure messages."""
    return f"{f} weights, {kv} cache, {'log-probabilities' if lp else 'plain'}"
