"""-m gpu: LLama2Model::generate() through `kuiper_decode --generate N --stop X [--then K]`.
(File name: sorts after the host suite, whose build it uses.)

generate() runs the prompt, then kllm_decoder_generate_until: its ids are those of the C-ABI decoder doing the
same calls (Decoder.prompt(), or the batched prefill plus one step with KUIPER_BATCHED_PREFILL=1, then
generate_until with the same stop id), greedy and sampled.  K more predict() steps after generate() continue
the same sequence, which pins the model's bookkeeping of the decoder's rows after generate()."""
import os
import subprocess

import numpy as np
import pytest

from test_z_host_cpp import ensure_built

pytestmark = pytest.mark.gpu

N, THEN = 40, 6


@pytest.mark.parametrize("sampled", [None, (0.8, 40, 5)])
@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("key,variant,family,prec", [("small", "llama2", "llama", "fp32"),
                                                     ("small-int8", "llama2", "llama", "int8"),
                                                     ("small-qwen", "qwen2", "qwen", "fp32")])
def test_cpp_generate_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec, batched, sampled):
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = SHAPES[key]
    w = synth_weights(shape, "cuda", 77)
    path = tmp_path / f"{key}.bin"
    write_checkpoint(str(path), shape, w)
    rng = np.random.default_rng(3)
    prompt = [1] + [int(t) for t in rng.integers(2, shape.vocab_size, 11)]
    n = len(prompt)
    dec = Decoder(shape, w)
    if sampled:
        dec.set_sampling(*sampled)

    def first_id():
        if batched:  # as the C++ model: all but the last prompt token batched, the last one stepped
            (dec.prefill_w8 if shape.group_size else dec.prefill_tf32)(prompt[:-1])
            return dec.step(prompt[-1], n - 1)
        return dec.prompt(prompt)

    first = first_id()
    probe = [first] + dec.generate_until(first, n, N - 1 + THEN)  # the uninterrupted sequence
    j = max(j for j in range(N - 5) if probe[j] not in probe[:j])  # a stop partway, where the sequence allows
    stop = probe[j]
    first_id()
    got = [first] if first == stop else [first] + dec.generate_until(first, n, N - 1, [stop])
    assert got == probe[:j + 1]
    dec.close()

    env = dict(os.environ)
    if batched:
        env["KUIPER_BATCHED_PREFILL"] = "1"
    if sampled:
        env.update(KUIPER_TEMPERATURE=str(sampled[0]), KUIPER_TOP_K=str(sampled[1]), KUIPER_SEED=str(sampled[2]))
    cmd = [str(ensure_built(variant)), str(path), family, prec, "1", *map(str, prompt), "--generate", str(N)]
    # two stop ids: the first one that occurs ends the run
    other = shape.vocab_size - 1 if stop != shape.vocab_size - 1 else 0
    r = subprocess.run(cmd + ["--stop", str(other), "--stop", str(stop)], capture_output=True, text=True, timeout=300,
                       env=env)
    assert r.returncode == 0, r.stderr
    want = next(probe[:i + 1] for i in range(N) if probe[i] in (stop, other))
    assert [int(x) for x in r.stdout.split()] == want
    # no stop id within reach: all N ids; then K predict() steps continue the same sequence
    absent = next(t for t in range(shape.vocab_size) if t not in probe)
    r = subprocess.run(cmd + ["--stop", str(absent), "--then", str(THEN)], capture_output=True, text=True,
                       timeout=300, env=env)
    assert r.returncode == 0, r.stderr
    assert [int(x) for x in r.stdout.split()] == probe[:N + THEN]
    # stop, then continue with predict(): the stepped ids are the uninterrupted sequence's
    r = subprocess.run(cmd + ["--stop", str(stop), "--then", str(THEN)], capture_output=True, text=True,
                       timeout=300, env=env)
    assert r.returncode == 0, r.stderr
    assert [int(x) for x in r.stdout.split()] == probe[:j + 1 + THEN]
