"""-m gpu: the frequency and presence penalties and the logit bias in the C++ model, through KUIPER_FREQUENCY_PENALTY /
KUIPER_PRESENCE_PENALTY and kuiper_decode --frequency-presence F P [FROM] / --logit-bias ID:B,...  (File name: sorts
after the host suite, whose build it uses.)

kuiper_decode prints the same ids as the C-ABI decoder with the same settings on the fused path (predict() on
embedding rows) and on the layer path (--layers: SeededSampler's kllm_logit_penalties_f32 over the ids the tool fed),
greedy and sampled, and through LLama2Model::generate().  A bias id outside the vocabulary is refused once the decoder
exists (the other invalid settings: test_z_host_cpp_draw_settings.py)."""
import os
import subprocess

import pytest

from test_z_host_cpp import ensure_built, run_decode
from test_z_host_cpp_repetition_penalty import MODELS, checkpoint, ids_of

pytestmark = pytest.mark.gpu

# (T, top_k, top_p, seed, penalty, frequency, presence, from_pos, bias)
SETTINGS = [(0.0, 0, 1.0, 0, 1.0, 0.8, 1.5, 0, {}), (0.0, 0, 1.0, 0, 1.3, 0.0, 1.5, 4, {7: 2.5, 11: -3.0}),
            (0.7, 20, 0.8, 2**40 + 7, 1.05, 0.5, 0.5, 0, {3: 1.0}), (0.8, 0, 1.0, 3, 1.0, -0.3, 0.0, 2, {})]


def decoder(shape, w, T, k, p, seed, theta, f, pr, from_pos, bias):
    from kuiperllama_b200 import Decoder
    dec = Decoder(shape, w)
    if T > 0:
        dec.set_sampling(T, k, seed, top_p=p)
    dec.set_repetition_penalty(theta, 0)
    dec.set_frequency_presence(f, pr, from_pos)
    dec.set_logit_bias(bias)
    return dec


def flags(theta, f, pr, from_pos, bias):
    out = ["--repetition-penalty", str(theta), "0", "--frequency-presence", str(f), str(pr), str(from_pos)]
    if bias:
        out += ["--logit-bias", ",".join(f"{i}:{b}" for i, b in bias.items())]
    return out


def env_for(T, k, p, seed):
    env = dict(os.environ)
    if T > 0:
        env.update(KUIPER_TEMPERATURE=str(T), KUIPER_TOP_K=str(k), KUIPER_TOP_P=str(p), KUIPER_SEED=str(seed))
    return env


@pytest.mark.parametrize("key,variant,family,prec", MODELS)
@pytest.mark.parametrize("T,k,p,seed,theta,f,pr,from_pos,bias", SETTINGS)
def test_cpp_logit_penalties_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec, T, k, p, seed, theta,
                                               f, pr, from_pos, bias):
    shape, w, path = checkpoint(tmp_path, key)
    prompt, steps = [1, 5, 9, 5], 40
    dec = decoder(shape, w, T, k, p, seed, theta, f, pr, from_pos, bias)
    want, tok = [], None
    for pos in range(steps):
        tok = dec.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
        want.append(tok)
    want = want[len(prompt) - 1:]
    dec.close()
    for layers in (False, True):
        r = subprocess.run([str(ensure_built(variant)), str(path), family, prec, str(steps), *map(str, prompt),
                            *(["--layers"] if layers else []), *flags(theta, f, pr, from_pos, bias)],
                           capture_output=True, text=True, timeout=300, env=env_for(T, k, p, seed))
        assert ids_of(r)[len(prompt) - 1:] == want, ("layers" if layers else "fused")
    if f or pr:
        assert "frequency_penalty" in r.stderr  # init() logs the setting


@pytest.mark.parametrize("key,variant,family,prec", MODELS[:1])
def test_cpp_environment_and_generate(kllm_lib, tmp_path, key, variant, family, prec):
    T, k, p, seed = 0.7, 20, 0.8, 11
    shape, w, path = checkpoint(tmp_path, key)
    prompt = [1, 5, 9, 5, 3, 3]
    N = 30
    dec = decoder(shape, w, T, k, p, seed, 1.0, 0.4, 1.2, 0, {})
    first = dec.prompt(prompt)
    probe = [first] + dec.generate_until(first, len(prompt), N - 1)
    dec.close()
    env = dict(env_for(T, k, p, seed), KUIPER_FREQUENCY_PENALTY="0.4", KUIPER_PRESENCE_PENALTY="1.2")
    absent = next(t for t in range(shape.vocab_size) if t not in probe)
    r = subprocess.run([str(ensure_built(variant)), str(path), family, prec, "1", *map(str, prompt), "--generate",
                        str(N), "--stop", str(absent)], capture_output=True, text=True, timeout=300, env=env)
    assert ids_of(r) == probe[:N]


def test_cpp_refuses_a_bias_id_outside_the_vocabulary(kllm_lib, tmp_path):
    _, _, path = checkpoint(tmp_path, "small", "cpu")
    r = subprocess.run([str(ensure_built("llama2")), str(path), "llama", "fp32", "8", "1", "5", "--logit-bias",
                        "100000000:1"], capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "init failed" in r.stderr, (r.returncode, r.stderr)


def test_cpp_copy_at_is_refused_with_the_settings(kllm_lib, tmp_path):
    _, _, path = checkpoint(tmp_path, "small", "cpu")
    r = run_decode("llama2", path, "llama", "fp32", 12, [1, 5, 9], copy_at=6,
                   env=dict(os.environ, KUIPER_PRESENCE_PENALTY="1.5"))
    assert r.returncode != 0 and "presence" in r.stderr, (r.returncode, r.stderr)
