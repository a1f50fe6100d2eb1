"""The C++ model's bf16 weights (LLama2Model::set_bf16_weights, KUIPER_WEIGHTS, kuiper_decode --weights).
(File name: sorts after the host suite, whose build it uses.)

not gpu: the host's rounding (base::fp32_to_bf16_rne, through kuiper_selftest --bf16-round) equals torch.bfloat16 bit
         for bit on ties, subnormals, zeros, infinities, NaN, the largest finite values and a random sweep; init()
         refuses an invalid KUIPER_WEIGHTS, an int8 checkpoint and tensor parallelism, naming the setting, before it
         touches a device.
gpu:     on a checkpoint whose fp32 weights are already bf16 values, bf16 weights give the default fp32 run's ids and
         logits; on any checkpoint, the C-ABI bf16 decoder's over torch-rounded weights; init() then holds at least
         45 % of the fp32 matrix bytes less device memory; forward() (--layers) returns its error.
"""
import os
import subprocess
from dataclasses import replace

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from test_weights_bf16_rule import special_inputs
from test_z_host_cpp import build_host, ensure_built


def decode(path, n_steps, prompt, *flags, prec="fp32", logits=None, **env):
    cmd = [str(ensure_built("llama2")), str(path), "llama", prec, str(n_steps), *map(str, prompt), *flags]
    if logits is not None:
        cmd += ["--logits", str(logits)]
    return subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, **env))


def test_host_rounding_matches_torch_bfloat16(kllm_lib, tmp_path):
    ensure_built("llama2")
    x = special_inputs()
    src, dst = tmp_path / "in.f32", tmp_path / "out.u16"
    x.tofile(src)
    r = subprocess.run([str(build_host.binary("llama2", "kuiper_selftest")), "--bf16-round", str(src), str(dst)],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    got = np.fromfile(dst, dtype=np.uint16)
    want = torch.from_numpy(x.copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    nan = np.isnan(x)
    assert got.shape == want.shape
    assert np.array_equal(got[~nan], want[~nan])
    widened = (got.astype(np.uint32) << 16).view(np.float32)
    assert np.isnan(widened[nan]).all()  # NaN stays NaN
    assert np.array_equal(np.signbit(widened[nan]), np.signbit(x[nan]))


@pytest.mark.parametrize("case", ["env", "int8", "tp"])
def test_host_refuses_what_bf16_weights_cannot_run(kllm_lib, case):
    if case == "env":
        r = decode(GOLDEN / "tiny_llama2_fp32.bin", 4, [1], KUIPER_WEIGHTS="fp16")
        assert r.returncode != 0 and "KUIPER_WEIGHTS" in r.stderr, r.stderr
    elif case == "int8":
        for r in (decode(GOLDEN / "tiny_llama2_int8.bin", 4, [1], "--weights", "bf16", prec="int8"),
                  decode(GOLDEN / "tiny_llama2_int8.bin", 4, [1], prec="int8", KUIPER_WEIGHTS="bf16")):
            assert r.returncode != 0 and "init failed" in r.stderr and "fp32 checkpoints" in r.stderr, r.stderr
    else:
        r = decode(GOLDEN / "tiny_llama2_fp32.bin", 4, [1], "--weights", "bf16", KUIPER_TP_WORLD="2",
                   KUIPER_TP_RANK="0")
        assert r.returncode != 0 and "init failed" in r.stderr and "one GPU" in r.stderr, r.stderr


def ids_and_logits(r, path):
    assert r.returncode == 0, r.stderr
    return [int(t) for t in r.stdout.split()], np.fromfile(path, dtype=np.uint32)


def device_bytes(r):
    line = [x for x in r.stderr.splitlines() if x.startswith("device bytes after init:")]
    return int(line[-1].split(":")[1])


@pytest.mark.gpu
def test_bf16_representable_checkpoint_equals_the_fp32_run(kllm_lib, tmp_path):
    from kuiperllama_b200 import SHAPES, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    from kuiperllama_b200.decoder import bf16_weights, widen_weights
    shape = SHAPES["small"]
    w = widen_weights(bf16_weights(synth_weights(shape, "cuda", 11)))  # every matrix value is a bf16 value
    path = tmp_path / "w.bin"
    write_checkpoint(str(path), shape, w)
    prompt, n = [1, 5, 9, 30], 40
    a = ids_and_logits(decode(path, n, prompt, logits=tmp_path / "a.f32"), tmp_path / "a.f32")
    b = ids_and_logits(decode(path, n, prompt, "--weights", "bf16", logits=tmp_path / "b.f32"), tmp_path / "b.f32")
    c = ids_and_logits(decode(path, n, prompt, logits=tmp_path / "c.f32", KUIPER_WEIGHTS="bf16"), tmp_path / "c.f32")
    assert a[0] == b[0] == c[0]
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[1], c[1])


@pytest.mark.gpu
@pytest.mark.parametrize("key,shared", [("small", False), ("small", True)])
def test_bf16_weights_equal_the_cabi_bf16_decoder(kllm_lib, tmp_path, key, shared):
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    from kuiperllama_b200.decoder import bf16_weights
    shape = replace(SHAPES[key], shared_classifier=shared)
    w = synth_weights(shape, "cuda", 12)
    path = tmp_path / "w.bin"
    write_checkpoint(str(path), shape, w)
    prompt, n = [1, 5, 9], 40
    got = ids_and_logits(decode(path, n, prompt, "--weights", "bf16", logits=tmp_path / "l.f32"), tmp_path / "l.f32")
    dec = Decoder(shape, bf16_weights(w), weight_format="bf16")
    want, tok = [], None
    for pos in range(n):
        tok = dec.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
        want.append(tok)
    assert got[0][len(prompt) - 1:] == want[len(prompt) - 1:]
    assert np.array_equal(got[1], dec.logits().view(np.uint32))
    dec.close()
    r = decode(path, 8, prompt, "--weights", "bf16", "--layers")
    assert r.returncode != 0 and "no bf16 kernels" in r.stderr, r.stderr


@pytest.mark.gpu
def test_bf16_weights_hold_less_device_memory(kllm_lib, tmp_path):
    from kuiperllama_b200 import ModelShape, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = ModelShape("mem-fp32", 1024, 2816, 4, 8, 2, 8000, 128)
    w = synth_weights(shape, "cuda", 13)
    path = tmp_path / "w.bin"
    write_checkpoint(str(path), shape, w)
    del w
    torch.cuda.empty_cache()
    d, h, L, kv, V = shape.dim, shape.hidden_dim, shape.layer_num, shape.kv_dim, shape.vocab_size
    matrix_bytes = 4 * (L * (2 * d * d + 2 * kv * d + 3 * h * d) + V * d)
    f32 = device_bytes(decode(path, 4, [1, 2]))
    b16 = device_bytes(decode(path, 4, [1, 2], "--weights", "bf16"))
    print("[weights-bf16] C++ host device bytes after init:", f32, "fp32,", b16, "bf16; fp32 matrices", matrix_bytes,
          flush=True)
    assert f32 - b16 >= 0.45 * matrix_bytes, (f32, b16, matrix_bytes)
