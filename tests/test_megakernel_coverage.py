"""Without a GPU: every non-profiling kernel of the persistent engine's table (tests/megakernel_table.py) is run by at
least one GPU case that holds what it computes to a model -- the fp64 decode model for the plain kernels, the
log-probability mirror of the plain kernel's logits for the log-probability ones.  The cases are read from the GPU
modules' own lists, so a kernel added to the table without such a case, or a case list that loses a row's last case,
fails here."""
from decode_model_util import GEOMETRIES, weight_format_of
from megakernel_table import MODEL_CHECKED, row


def model_checked_runs():
    """{(weight format, KV cache, log-probabilities): [the GPU tests that run that kernel against a model]}."""
    import test_decode_model_gpu
    import test_kv_bf16_gpu
    import test_kv_fp8_gpu
    import test_logprobs_gpu
    import test_weights_bf16_gpu
    runs = {}

    def plain(key, weight_format, kv_cache, test):
        runs.setdefault((weight_format_of(GEOMETRIES[key], weight_format), kv_cache, False), []).append(test)

    for key, _, _ in test_decode_model_gpu.CASES:
        plain(key, "fp32", "fp32", "test_decode_model_gpu.py::test_decode_against_the_model")
    for key, _ in test_weights_bf16_gpu.BOUND_CASES:
        plain(key, "bf16", "fp32",
              "test_weights_bf16_gpu.py::test_fast_mode_at_its_own_geometry_within_the_model_bounds")
    for key, _, _, weight_format in test_kv_bf16_gpu.BF16_CASES:
        plain(key, weight_format, "bf16", "test_kv_bf16_gpu.py::test_bf16_decode_against_the_model")
    for key, _, _, _, weight_format in test_kv_fp8_gpu.FP8_CASES:
        plain(key, weight_format, "fp8", "test_kv_fp8_gpu.py::test_fp8_decode_against_the_model")
    for weight_format, kv_cache in test_logprobs_gpu.KERNEL_PAIRS:
        runs.setdefault((weight_format, kv_cache, True), []).append(
            "test_logprobs_gpu.py::test_kernel_pair_records_match_the_mirror")
    return runs


def test_every_megakernel_instantiation_runs_against_a_model():
    runs = model_checked_runs()
    missing = [row(*t) for t in MODEL_CHECKED if t not in runs]
    assert not missing, f"kernels without a model-checked GPU case: {missing}"
    unknown = sorted(set(runs) - set(MODEL_CHECKED))
    assert not unknown, f"GPU cases of kernels the table does not hold: {unknown}"
