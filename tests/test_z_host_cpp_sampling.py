"""-m gpu: seeded sampling in the C++ model through KUIPER_TEMPERATURE / KUIPER_TOP_K / KUIPER_SEED.
(File name: sorts after the host suite, whose greedy parity results it builds on.)

The demo loop through kuiper_decode prints the same ids as the C-ABI decoder with the same settings: on the
fused path, on the layer path (sampler::SeededSampler over kllm_sample_f32), through predict()'s own
forward + post_processing, and with the settings given by set_sampling() instead of the environment.  Without the variables the
host suite (tests/test_z_host_cpp.py) pins that nothing changed."""
import os
import subprocess

import pytest

from test_z_host_cpp import ensure_built, run_decode

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("key,variant,family,prec", [("small", "llama2", "llama", "fp32"),
                                                     ("small-int8", "llama2", "llama", "int8"),
                                                     ("small-qwen", "qwen2", "qwen", "fp32")])
@pytest.mark.parametrize("T,k,seed", [(0.8, 0, 3), (0.9, 40, 2**40 + 7)])
def test_cpp_sampling_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec, T, k, seed):
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = SHAPES[key]
    w = synth_weights(shape, "cuda", 77)
    path = tmp_path / f"{key}.bin"
    write_checkpoint(str(path), shape, w)
    prompt, steps = [1, 5, 9], 40
    dec = Decoder(shape, w)
    dec.set_sampling(T, k, seed)
    want, tok = [], None
    for pos in range(steps):
        tok = dec.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
        want.append(tok)
    want = want[len(prompt) - 1:]
    dec.close()
    env = dict(os.environ, KUIPER_TEMPERATURE=str(T), KUIPER_TOP_K=str(k), KUIPER_SEED=str(seed))
    for layers in (False, True):
        r = run_decode(variant, path, family, prec, steps, prompt, layers=layers, env=env)
        assert r.returncode == 0, r.stderr
        chosen = [int(x) for x in r.stdout.split()]
        assert chosen[len(prompt) - 1:] == want, ("layers" if layers else "fused")
    # a step handed a COPY of its embedding row goes predict -> forward -> post_processing (the model's own
    # SeededSampler, given the position there); the explicit set_sampling() API draws the same ids
    r = run_decode(variant, path, family, prec, steps, prompt, env=env, copy_at=len(prompt) + 4)
    assert r.returncode == 0, r.stderr
    assert [int(x) for x in r.stdout.split()][len(prompt) - 1:] == want, "copy-at"
    r = subprocess.run([str(ensure_built(variant)), str(path), family, prec, str(steps), *map(str, prompt),
                        "--copy-at", str(len(prompt) + 7), "--sampling", str(T), str(k), str(seed)],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    assert [int(x) for x in r.stdout.split()][len(prompt) - 1:] == want, "set_sampling"
    greedy = run_decode(variant, path, family, prec, steps, prompt)
    assert greedy.returncode == 0 and greedy.stdout.split() != r.stdout.split()
