"""-m gpu: the repetition penalty in the C++ model through KUIPER_REPETITION_PENALTY / KUIPER_REPEAT_LAST_N and
kuiper_decode --repetition-penalty P N.  (File name: sorts after the host suite, whose build it uses.)

kuiper_decode prints the same ids as the C-ABI decoder with the same settings: on the fused path (predict() on
embedding rows), on the layer path (--layers: SeededSampler's kllm_repetition_penalty_f32 over the ids the tool
fed) and through LLama2Model::generate() (with and without the batched prefill).  predict()
of a tensor that is not an embedding() row (--copy-at) is refused while the penalty is on.  (Invalid settings:
test_z_host_cpp_draw_settings.py.)"""
import os
import subprocess

import numpy as np
import pytest

from test_z_host_cpp import ensure_built, run_decode

pytestmark = pytest.mark.gpu

MODELS = [("small", "llama2", "llama", "fp32"), ("small-int8", "llama2", "llama", "int8"),
          ("small-qwen", "qwen2", "qwen", "fp32")]
# (T, top_k, top_p, seed, penalty, last_n): greedy, and Qwen2.5-Instruct's config with a window
SETTINGS = [(0.0, 0, 1.0, 0, 1.3, 0), (0.7, 20, 0.8, 2**40 + 7, 1.05, 0), (0.8, 0, 1.0, 3, 1.5, 8)]


def checkpoint(tmp_path, key, device="cuda"):
    from kuiperllama_b200 import SHAPES, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = SHAPES[key]
    w = synth_weights(shape, device, 77)
    path = tmp_path / f"{key}.bin"
    write_checkpoint(str(path), shape, w)
    return shape, w, path


def decoder(shape, w, T, k, p, seed, theta, last_n):
    from kuiperllama_b200 import Decoder
    dec = Decoder(shape, w)
    if T > 0:
        dec.set_sampling(T, k, seed, top_p=p)
    dec.set_repetition_penalty(theta, last_n)
    return dec


def env_for(T, k, p, seed, theta, last_n, **extra):
    env = dict(os.environ, KUIPER_REPETITION_PENALTY=str(theta), KUIPER_REPEAT_LAST_N=str(last_n), **extra)
    if T > 0:
        env.update(KUIPER_TEMPERATURE=str(T), KUIPER_TOP_K=str(k), KUIPER_TOP_P=str(p), KUIPER_SEED=str(seed))
    return env


def ids_of(r):
    assert r.returncode == 0, r.stderr
    return [int(x) for x in r.stdout.split()]


@pytest.mark.parametrize("key,variant,family,prec", MODELS)
@pytest.mark.parametrize("T,k,p,seed,theta,last_n", SETTINGS)
def test_cpp_penalty_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec, T, k, p, seed, theta, last_n):
    shape, w, path = checkpoint(tmp_path, key)
    prompt, steps = [1, 5, 9, 5], 40
    dec = decoder(shape, w, T, k, p, seed, theta, last_n)
    want, tok = [], None
    for pos in range(steps):
        tok = dec.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
        want.append(tok)
    want = want[len(prompt) - 1:]
    dec.close()
    plain = decoder(shape, w, T, k, p, seed, 1.0, 0)
    tok, unpenalised = None, []
    for pos in range(steps):
        tok = plain.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
        unpenalised.append(tok)
    plain.close()
    if T == 0:  # (sampling over these flat synthetic logits may draw the same ids either way)
        assert unpenalised[len(prompt) - 1:] != want, "the penalty must change these ids"
    env = env_for(T, k, p, seed, theta, last_n)
    for layers in (False, True):
        r = run_decode(variant, path, family, prec, steps, prompt, layers=layers, env=env)
        assert ids_of(r)[len(prompt) - 1:] == want, ("layers" if layers else "fused")
    assert "repetition_penalty" in r.stderr  # init() logs the setting
    # --repetition-penalty (LLama2Model::set_repetition_penalty) instead of the environment, which it overrides
    bad = dict(env, KUIPER_REPETITION_PENALTY="2.5", KUIPER_REPEAT_LAST_N="3")
    for extra in ([], ["--layers"]):
        r = subprocess.run([str(ensure_built(variant)), str(path), family, prec, str(steps), *map(str, prompt), *extra,
                            "--repetition-penalty", str(theta), str(last_n)],
                           capture_output=True, text=True, timeout=300, env=bad)
        assert ids_of(r)[len(prompt) - 1:] == want, ("--repetition-penalty", extra)


@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("key,variant,family,prec", MODELS)
def test_cpp_generate_with_penalty_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec, batched):
    T, k, p, seed, theta, last_n = SETTINGS[1]
    shape, w, path = checkpoint(tmp_path, key)
    rng = np.random.default_rng(3)
    prompt = [1] + [int(t) for t in rng.integers(2, shape.vocab_size, 11)]
    n, N, THEN = len(prompt), 40, 6
    dec = decoder(shape, w, T, k, p, seed, theta, last_n)
    if batched:  # as the C++ model: all but the last prompt token batched, the last one stepped
        (dec.prefill_w8 if shape.group_size else dec.prefill_tf32)(prompt[:-1])
        first = dec.step(prompt[-1], n - 1)
    else:
        first = dec.prompt(prompt)
    probe = [first] + dec.generate_until(first, n, N - 1 + THEN)
    dec.close()
    env = env_for(T, k, p, seed, theta, last_n)
    if batched:
        env["KUIPER_BATCHED_PREFILL"] = "1"
    absent = next(t for t in range(shape.vocab_size) if t not in probe)
    r = subprocess.run([str(ensure_built(variant)), str(path), family, prec, "1", *map(str, prompt), "--generate",
                        str(N), "--stop", str(absent), "--then", str(THEN)],
                       capture_output=True, text=True, timeout=300, env=env)
    assert ids_of(r) == probe[:N + THEN]


def test_cpp_copy_at_is_refused_with_the_penalty(kllm_lib, tmp_path):
    _, _, path = checkpoint(tmp_path, "small", "cpu")
    r = run_decode("llama2", path, "llama", "fp32", 12, [1, 5, 9], copy_at=6,
                   env=dict(os.environ, KUIPER_REPETITION_PENALTY="1.3"))
    assert r.returncode != 0 and "repetition_penalty" in r.stderr, (r.returncode, r.stderr)
    # penalty 1 is off: the same call runs
    r = run_decode("llama2", path, "llama", "fp32", 12, [1, 5, 9], copy_at=6,
                   env=dict(os.environ, KUIPER_REPETITION_PENALTY="1"))
    assert r.returncode == 0, r.stderr
