"""-m gpu: nucleus (top-p) sampling in the C++ model through KUIPER_TOP_P and kuiper_decode --top-p.
(File name: sorts after the host suite, whose greedy parity results it builds on.)

kuiper_decode prints the same ids as the C-ABI decoder with the same settings: on the fused path, on the
layer path (sampler::SeededSampler over kllm_sample_top_p_f32) and through predict()'s own forward +
post_processing (--copy-at), with the setting from the environment and from LLama2Model::set_top_p()."""
import os
import subprocess

import pytest

from test_z_host_cpp import ensure_built, run_decode

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("key,variant,family,prec", [("small", "llama2", "llama", "fp32"),
                                                     ("small-int8", "llama2", "llama", "int8"),
                                                     ("small-qwen", "qwen2", "qwen", "fp32")])
@pytest.mark.parametrize("T,k,p,seed", [(0.8, 0, 0.9, 3), (0.7, 20, 0.8, 2**40 + 7)])
def test_cpp_top_p_identical_to_cabi(kllm_lib, tmp_path, key, variant, family, prec, T, k, p, seed):
    from kuiperllama_b200 import SHAPES, Decoder, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = SHAPES[key]
    w = synth_weights(shape, "cuda", 77)
    path = tmp_path / f"{key}.bin"
    write_checkpoint(str(path), shape, w)
    prompt, steps = [1, 5, 9], 40
    dec = Decoder(shape, w)
    dec.set_sampling(T, k, seed, top_p=p)
    want, tok = [], None
    for pos in range(steps):
        tok = dec.step(prompt[pos] if pos < len(prompt) else tok, pos, pos < len(prompt) - 1)
        want.append(tok)
    want = want[len(prompt) - 1:]
    dec.close()
    env = dict(os.environ, KUIPER_TEMPERATURE=str(T), KUIPER_TOP_K=str(k), KUIPER_SEED=str(seed), KUIPER_TOP_P=str(p))
    for layers in (False, True):
        r = run_decode(variant, path, family, prec, steps, prompt, layers=layers, env=env)
        assert r.returncode == 0, r.stderr
        assert [int(x) for x in r.stdout.split()][len(prompt) - 1:] == want, ("layers" if layers else "fused")
    r = run_decode(variant, path, family, prec, steps, prompt, env=env, copy_at=len(prompt) + 4)
    assert r.returncode == 0, r.stderr
    assert [int(x) for x in r.stdout.split()][len(prompt) - 1:] == want, "copy-at"
    # --top-p (LLama2Model::set_top_p) instead of the environment, which it overrides
    bad_env = dict(os.environ, KUIPER_TOP_P="0.5")
    for extra in ([], ["--layers"], ["--copy-at", str(len(prompt) + 7)]):
        r = subprocess.run([str(ensure_built(variant)), str(path), family, prec, str(steps), *map(str, prompt), *extra,
                            "--sampling", str(T), str(k), str(seed), "--top-p", str(p)],
                           capture_output=True, text=True, timeout=300, env=bad_env)
        assert r.returncode == 0, r.stderr
        assert [int(x) for x in r.stdout.split()][len(prompt) - 1:] == want, ("--top-p", extra)
    assert "top_p" in r.stderr  # init() logs the setting
