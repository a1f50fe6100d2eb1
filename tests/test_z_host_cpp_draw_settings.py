"""The C++ model's refusals of invalid draw settings, through kuiper_decode.  (File name: sorts after the host suite,
whose build it uses.)

init() validates the settings before it touches a CUDA device, so these run without a GPU: each invalid value, from
the environment and from its kuiper_decode flag (the LLama2Model setter), fails init() with an error that names it.
Without a GPU init() fails in any case, so every check also looks for the setting's name in the error.  A bias id
outside the vocabulary is refused by the decoder once CUDA is up, so that case stays with the GPU tests
(test_z_host_cpp_logit_penalties.py)."""
import os
import subprocess

import pytest

from conftest import GOLDEN
from test_z_host_cpp import ensure_built


def decode(*flags, **env):
    return subprocess.run([str(ensure_built("llama2")), str(GOLDEN / "tiny_llama2_fp32.bin"), "llama", "fp32", "8",
                           "1", "5", *flags], capture_output=True, text=True, timeout=300, env=dict(os.environ, **env))


@pytest.mark.parametrize("value", ["-0.5", "nan"])
def test_cpp_refuses_invalid_temperature(kllm_lib, value):
    for r in (decode(KUIPER_TEMPERATURE=value), decode("--sampling", value, "0", "1")):
        assert r.returncode != 0 and "temperature" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.parametrize("value", ["0", "-0.5", "1.5", "nan"])
def test_cpp_refuses_invalid_top_p(kllm_lib, value):
    for r in (decode(KUIPER_TEMPERATURE="0.8", KUIPER_TOP_P=value),
              decode("--sampling", "0.8", "0", "1", "--top-p", value)):
        assert r.returncode != 0 and "top_p" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.parametrize("value,last_n", [("0", "0"), ("-1.1", "0"), ("nan", "0"), ("inf", "0"), ("1.2", "-1")])
def test_cpp_refuses_invalid_penalty(kllm_lib, value, last_n):
    for r in (decode(KUIPER_REPETITION_PENALTY=value, KUIPER_REPEAT_LAST_N=last_n),
              decode("--repetition-penalty", value, last_n)):
        assert r.returncode != 0 and "repetition_penalty" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.parametrize("args", [["--frequency-presence", "nan", "0"], ["--frequency-presence", "0", "inf"],
                                  ["--frequency-presence", "0.5", "0", "-1"], ["--logit-bias", "3:1,3:2"],
                                  ["--logit-bias", "3:nan"], ["--logit-bias", "3:inf"], ["--logit-bias", "-1:1"]])
def test_cpp_refuses_invalid_settings(kllm_lib, args):
    r = decode(*args)
    named = "logit bias" if args[0] == "--logit-bias" else "presence"
    assert r.returncode != 0 and "init failed" in r.stderr and named in r.stderr, (r.returncode, r.stderr)


@pytest.mark.parametrize("var", ["KUIPER_FREQUENCY_PENALTY", "KUIPER_PRESENCE_PENALTY"])
def test_cpp_refuses_invalid_frequency_presence_from_the_environment(kllm_lib, var):
    r = decode(**{var: "nan"})
    assert r.returncode != 0 and "init failed" in r.stderr and "presence" in r.stderr, (r.returncode, r.stderr)


def test_cpp_refuses_invalid_top_n(kllm_lib):
    for bad in ("21", "-2"):
        r = decode("--logprobs", bad)
        assert r.returncode != 0 and "logprobs" in r.stderr, (bad, r.returncode, r.stderr)
