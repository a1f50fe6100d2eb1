"""-m gpu: the C++ model's opt-in batched prompt prefill (KUIPER_BATCHED_PREFILL=1, LLama2Model::set_batched_prefill).
(File name: sorts after the decoder and host suites, whose parity results it builds on.)

With the switch on, the demo loop's first prompt row runs every prompt position but the last through
kllm_decoder_prefill_w8 / _tf32, and the last prompt row and everything after it step through the fused decoder.
The C-ABI decoder doing the same calls runs the same deterministic kernels, so ids and logits are bit-identical.
Without the switch the host suite (tests/test_z_host_cpp.py) pins that nothing changed."""
import os

import numpy as np
import pytest

from test_z_host_cpp import run_decode

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("key,prec", [("small-int8", "int8"), ("small", "fp32")])
def test_cpp_batched_prefill_switch_identical_to_cabi(kllm_lib, tmp_path, key, prec):
    """A 70-token prompt plus 20 free-running steps through the C++ model with KUIPER_BATCHED_PREFILL=1 == the
    C-ABI decoder prefilled over prompt[:-1] and stepped from the last prompt position on.  A step inside the
    prefilled range that leaves the fused decoder (--copy-at) changes neither ids nor final logits."""
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = SHAPES[key]
    w = synth_weights(shape, "cuda", 77)
    path = tmp_path / f"{key}.bin"
    write_checkpoint(str(path), shape, w)
    rng = np.random.default_rng(12)
    prompt = [1] + [int(t) for t in rng.integers(2, shape.vocab_size, 69)]
    n = len(prompt) + 20
    dec = Decoder(shape, w)
    (dec.prefill_w8 if shape.group_size else dec.prefill_tf32)(prompt[:-1])
    tok = dec.step(prompt[-1], len(prompt) - 1)
    want = [tok]
    for pos in range(len(prompt), n):
        tok = dec.step(tok, pos)
        want.append(tok)
    env = dict(os.environ, KUIPER_BATCHED_PREFILL="1")
    a, b = tmp_path / "a.f32", tmp_path / "b.f32"
    r = run_decode("llama2", path, "llama", prec, n, prompt, logits=a, env=env)
    assert r.returncode == 0, r.stderr
    chosen = [int(x) for x in r.stdout.split()]
    assert chosen[:len(prompt) - 1] == [-1] * (len(prompt) - 1)
    assert chosen[len(prompt) - 1:] == want
    assert np.array_equal(np.fromfile(a, dtype=np.uint32), dec.logits().view(np.uint32))
    dec.close()
    r1 = run_decode("llama2", path, "llama", prec, n, prompt, logits=b, env=env, copy_at=30)
    assert r1.returncode == 0, r1.stderr
    assert r1.stdout.split() == r.stdout.split()
    assert np.array_equal(np.fromfile(a, dtype=np.uint32), np.fromfile(b, dtype=np.uint32))
