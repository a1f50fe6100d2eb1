"""The fp8 KV cache's description rules and kernels, without a GPU.

1. kllm_decoder_create's refusals of an fp8 description (kllm_b200.h, kllm_decoder_desc::kv_cache / kv_scales): the
   fp8 cache without scales, a scale that is not finite and > 0, scales with another cache, tensor parallelism and
   the graph engine.  They come
   before the device lookup, so each returns its code on any machine.
2. The descriptor's new trailing field matches the header's layout.
(test_abi.py gates the fp8 cache's megakernel instantiations with every other one.)
"""
import ctypes
import subprocess

import pytest

from test_decoder_desc_refusals import E_INVALID, E_NODEVICE, E_UNSUPPORTED, L, _device_visible, _tp, create, valid_desc

from kuiperllama_b200 import HEADER_PATH, DecoderDesc

KVH = 2  # valid_desc's kv_head_num
_keep = []


def with_scales(d, values):
    arr = (ctypes.c_float * len(values))(*values)
    _keep.append(arr)
    d.kv_scales = ctypes.cast(arr, ctypes.POINTER(ctypes.c_float))


def fp8(d, scales=None):
    d.kv_cache = 2
    if scales is not None:
        with_scales(d, scales)


ONES = [1.0] * (2 * L * KVH)


@pytest.mark.parametrize("bad", [0.0, -0.0, -2.0, float("nan"), float("inf"), float("-inf")])
@pytest.mark.parametrize("at", [0, 2 * L * KVH - 1])
def test_a_bad_scale_is_invalid(kllm_lib, bad, at):
    d = valid_desc()
    s = list(ONES)
    s[at] = bad
    fp8(d, s)
    assert create(kllm_lib, d) == E_INVALID


@pytest.mark.parametrize("tp", [1, 2])
def test_fp8_cache_without_scales_is_invalid(kllm_lib, tp):
    """kv_cache 2 with kv_scales NULL: what a description written before the fp8 cache existed holds (its value 2 was
    refused then), refused before any rule of the cache itself."""
    d = valid_desc()
    if tp > 1:
        _tp(tp)(d)
    fp8(d)
    assert create(kllm_lib, d) == E_INVALID


@pytest.mark.parametrize("cache", [0, 1])
def test_scales_with_another_cache_are_invalid(kllm_lib, cache):
    d = valid_desc()
    d.kv_cache = cache
    with_scales(d, ONES)
    assert create(kllm_lib, d) == E_INVALID


def test_invalid_scales_come_before_tensor_parallelism(kllm_lib):
    d = valid_desc()
    _tp(2)(d)
    fp8(d, [0.0] + ONES[1:])
    assert create(kllm_lib, d) == E_INVALID


def test_fp8_cache_under_tensor_parallelism_is_unsupported(kllm_lib):
    d = valid_desc()
    _tp(2)(d)
    fp8(d, ONES)
    assert create(kllm_lib, d) == E_UNSUPPORTED


def test_fp8_cache_on_the_graph_engine_is_refused(kllm_lib, monkeypatch):
    monkeypatch.setenv("KLLM_ENGINE", "graph")
    d = valid_desc()
    fp8(d, ONES)
    assert create(kllm_lib, d) == E_UNSUPPORTED


@pytest.mark.parametrize("group_size,weights,scales", [(0, 0, ONES), (64, 0, ONES), (0, 1, ONES),
                                                        (0, 0, [0.5, 2.0, 1e-3, 3e4] * L)])
def test_valid_fp8_description_reaches_the_device_lookup(kllm_lib, group_size, weights, scales):
    if _device_visible():
        pytest.skip("a device is present: the description's fake pointers must not reach it")
    d = valid_desc(group_size)
    d.weights = weights
    fp8(d, scales)
    assert create(kllm_lib, d) == E_NODEVICE


def test_descriptor_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text(f'#include <stddef.h>\n#include <stdio.h>\n#include "{HEADER_PATH}"\n'
                   'int main(void) { printf("%zu %zu %d\\n", sizeof(kllm_decoder_desc), '
                   'offsetof(kllm_decoder_desc, kv_scales), KLLM_KV_FP8); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run(["cc", str(src), "-o", str(exe)], check=True)
    size, off, fp8_value = map(int, subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    assert (size, off, fp8_value) == (ctypes.sizeof(DecoderDesc), DecoderDesc.kv_scales.offset, 2)
    assert not DecoderDesc().kv_scales  # a zeroed struct: unit scales

