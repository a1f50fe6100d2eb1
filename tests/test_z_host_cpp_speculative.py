"""The C++ model's speculative decoding (LLama2Model::set_speculative, KUIPER_SPECULATIVE, kuiper_decode --speculative).
(File name: sorts after the host suite, whose build it uses.)

not gpu: init() refuses the fast numerics, tensor parallelism and values outside the ranges, naming the setting,
         before it touches a device.
gpu:     `kuiper_decode --generate N --speculative K` and KUIPER_SPECULATIVE=K print the ids of the run without it, on
         a repetitive prompt (whose drafts are accepted) and on plain ones, greedy and sampled, with a stop id.
"""
import os
import subprocess
from dataclasses import replace

import pytest

from conftest import GOLDEN
from test_z_host_cpp import ensure_built


def decode(path, n_steps, prompt, *flags, prec="fp32", **env):
    cmd = [str(ensure_built("llama2")), str(path), "llama", prec, str(n_steps), *map(str, prompt), *flags]
    return subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, **env))


@pytest.mark.parametrize("case", ["fast-flag", "fast-env", "tp", "range", "env"])
def test_host_refuses_what_speculative_decoding_cannot_run(kllm_lib, case):
    path = GOLDEN / "tiny_llama2_fp32.bin"
    if case == "fast-flag":
        r = decode(path, 1, [1], "--generate", "4", "--speculative", "2", KUIPER_NUMERICS="fast")
        want = "exact numerics"
    elif case == "fast-env":
        r = decode(path, 1, [1], "--generate", "4", KUIPER_NUMERICS="fast", KUIPER_SPECULATIVE="3")
        want = "exact numerics"
    elif case == "tp":
        r = decode(path, 1, [1], "--speculative", "2", KUIPER_TP_WORLD="2", KUIPER_TP_RANK="0")
        want = "one GPU"
    elif case == "range":
        r = decode(path, 1, [1], "--speculative", "8")
        want = "draft_len"
    else:
        r = decode(path, 1, [1], KUIPER_SPECULATIVE="four")
        want = "KUIPER_SPECULATIVE"
    assert r.returncode != 0 and "init failed" in r.stderr and want in r.stderr, r.stderr


def ids(r):
    assert r.returncode == 0, r.stderr
    return [int(t) for t in r.stdout.split()]


@pytest.mark.gpu
@pytest.mark.parametrize("sampled", [False, True])
def test_speculative_generate_prints_the_same_ids(kllm_lib, tmp_path, sampled):
    from kuiperllama_b200 import SHAPES, synth_weights
    from kuiperllama_b200.checkpoint import write_checkpoint
    shape = replace(SHAPES["small"], seq_len=160)
    path = tmp_path / "small.bin"
    write_checkpoint(str(path), shape, synth_weights(shape, "cpu", 11))
    env = dict(KUIPER_TEMPERATURE="0.9", KUIPER_TOP_K="40", KUIPER_SEED="7") if sampled else {}
    prompts = [[7, 8, 9, 10, 7, 8, 9, 10, 7, 8], [1, 2, 3], [5]]
    for prompt in prompts:
        plain = ids(decode(path, 1, prompt, "--generate", "100", **env))
        for k in (1, 3, 7):
            assert ids(decode(path, 1, prompt, "--generate", "100", "--speculative", str(k), **env)) == plain, k
        assert ids(decode(path, 1, prompt, "--generate", "100", KUIPER_SPECULATIVE="4", **env)) == plain
        # a stop id in the middle of the run
        stop = plain[len(plain) // 2]
        cut = plain[:plain.index(stop) + 1]
        assert ids(decode(path, 1, prompt, "--generate", "100", "--stop", str(stop), "--speculative", "4",
                          **env)) == cut
