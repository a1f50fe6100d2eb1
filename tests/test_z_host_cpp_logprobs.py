"""-m gpu: log-probabilities in the C++ model (LLama2Model::set_logprobs / logprobs / score) through
kuiper_decode --logprobs N and --score.  (File name: sorts after the host suite, whose build it uses.)

kuiper_decode prints what the C ABI returns, bit for bit: the record entries of a decode with the same settings, and
the scored log-probabilities of the same ids.  --layers with either is refused."""
import subprocess

import numpy as np
import pytest

from test_z_host_cpp import ensure_built

pytestmark = pytest.mark.gpu

MODELS = [("small", "llama2", "llama", "fp32"), ("small-int8", "llama2", "llama", "int8"),
          ("small-qwen", "qwen2", "qwen", "fp32")]


def checkpoint(tmp_path, key, device="cuda"):
    from kuiperllama_b200 import SHAPES, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = SHAPES[key]
    w = synth_weights(shape, device, 77)
    path = tmp_path / f"{key}.bin"
    write_checkpoint(str(path), shape, w)
    return shape, w, path


def decode(variant, path, family, prec, steps, ids, *extra):
    r = subprocess.run([str(ensure_built(variant)), str(path), family, prec, str(steps), *map(str, ids), *extra],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return r.stdout.splitlines()


def f32(s):
    return np.float32(float(s))


@pytest.mark.parametrize("key,variant,family,prec", MODELS)
@pytest.mark.parametrize("top_n", [0, 5])
def test_cpp_logprobs_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec, top_n):
    from kuiperllama_b200 import Decoder
    shape, w, path = checkpoint(tmp_path, key)
    prompt, steps = [1, 5, 9, 5], 24
    dec = Decoder(shape, w)
    dec.set_logprobs(top_n)
    tok = None
    for pos in range(steps):
        tok = dec.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
    ids, lp, ti, tl = dec.logprobs(0, steps)
    dec.close()
    lines = decode(variant, path, family, prec, steps, prompt, "--logprobs", str(top_n))
    rows = [l.split() for l in lines[1:]]
    assert [int(r[1]) for r in rows] == [p for p in range(steps) if ids[p] >= 0]
    assert len(rows) == steps - len(prompt) + 1  # the prompt positions before the last have no entry
    for r in rows:
        p = int(r[1])
        assert int(r[2]) == ids[p] and f32(r[3]).view(np.uint32) == lp[p].view(np.uint32), (key, p)
        assert len(r) == 4 + 2 * top_n
        for j in range(top_n):
            assert int(r[4 + 2 * j]) == ti[p, j] and f32(r[5 + 2 * j]).view(np.uint32) == tl[p, j].view(np.uint32)


@pytest.mark.parametrize("key,variant,family,prec", MODELS)
def test_cpp_score_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec):
    from kuiperllama_b200 import Decoder
    shape, w, path = checkpoint(tmp_path, key)
    tokens = [int(t) for t in np.random.default_rng(6).integers(0, shape.vocab_size, 40)]
    dec = Decoder(shape, w)
    want = dec.score(tokens)
    dec.close()
    lines = decode(variant, path, family, prec, 1, tokens, "--score")
    got = np.array([f32(x) for x in lines[0].split()], np.float32)
    assert (got.view(np.uint32) == want.view(np.uint32)).all()
    ppl = float(lines[1].split()[1])
    assert ppl == pytest.approx(float(np.exp(-np.mean(want.astype(np.float64)))), rel=1e-6)


def test_cpp_layers_refuses_logprobs(kllm_lib, tmp_path):
    _, _, path = checkpoint(tmp_path, "small", "cpu")
    for extra in (["--logprobs", "3"], ["--score"]):
        r = subprocess.run([str(ensure_built("llama2")), str(path), "llama", "fp32", "8", "1", "5", "--layers", *extra],
                           capture_output=True, text=True, timeout=300)
        assert r.returncode != 0 and "--layers" in r.stderr, (extra, r.returncode, r.stderr)
