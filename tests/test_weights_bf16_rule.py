"""bf16 weights (kllm_decoder_desc::weights = KLLM_WEIGHTS_BF16) without a GPU: the rounding rule of the Python helper,
the descriptor's layout against the header and the byte count.  tests/test_abi.py gates the persistent kernel's bf16
instantiations with every other one."""
import shutil
import subprocess

import numpy as np
import pytest
import torch

from kuiperllama_b200 import HEADER_PATH, SHAPES, DecoderDesc
from kuiperllama_b200.decoder import MATRICES, bf16_weights, widen_weights


def rne_bf16_bits(x):
    """Round to nearest even of fp32 values to bf16 bit patterns, written out on the integer bits: NaN stays a
    (quiet) NaN, everything else rounds by adding 0x7fff plus the lowest kept bit (finite values past the largest
    bf16 become inf)."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    nan = np.isnan(np.asarray(x, np.float32))
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    r[nan] = ((u[nan] >> 16) | 0x40).astype(np.uint16)
    return r


def special_inputs():
    f = np.float32
    ties = [0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,  # exact ties: to even, both directions, both signs
            0x3F808001, 0x3F817FFF, 0x00008000, 0x00018000]  # just past / below a tie; subnormal ties
    subn = [0x00000001, 0x00007FFF, 0x00010000, 0x007FFFFF, 0x807FFFFF, 0x80000001]
    big = [0x7F7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0xFF7FFFFF, 0xFF7F8000]  # the largest finite values: up to inf or not
    spec = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FBFFFFF]
    bits = np.array(ties + subn + big + spec, np.uint32)
    rng = np.random.default_rng(5)
    sweep = rng.integers(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32)
    return np.concatenate([bits, sweep]).view(f)


def test_helper_rounds_as_torch_bfloat16():
    x = special_inputs()
    t = torch.from_numpy(x.copy())
    want = t.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    w = {n: t.reshape(1, 1, -1) for n in MATRICES}
    w.update(tok_emb=t.reshape(1, -1), wcls=None)
    got = bf16_weights(w)
    for n in MATRICES + ("wcls",):
        assert got[n].dtype == torch.bfloat16
        g = got[n].reshape(-1).view(torch.int16).numpy().view(np.uint16)
        nan = np.isnan(x)
        assert np.array_equal(g[~nan], want[~nan]), n
        assert np.isnan(got[n].reshape(-1).float().numpy()[nan]).all(), n  # NaN stays NaN
    # the rule written out agrees with torch on every non-NaN input (the specials above included)
    mine = rne_bf16_bits(x)
    nan = np.isnan(x)
    assert np.array_equal(mine[~nan], want[~nan])
    # the largest finite fp32 values round up to inf, ties go to even
    assert np.isinf(got["wq"].float().numpy().reshape(-1)[np.where(x == np.float32(3.4028235e38))[0]]).all()
    assert got["wq"].reshape(-1)[0].item() == 1.0 and got["wq"].reshape(-1)[1].item() == 1.015625
    # the shared classifier becomes a separate bf16 copy of the embedding; the embedding stays fp32
    assert got["tok_emb"] is w["tok_emb"] and got["tok_emb"].dtype == torch.float32
    wide = widen_weights(got)
    for n in MATRICES + ("wcls",):
        assert wide[n].dtype == torch.float32
        assert torch.equal(wide[n].to(torch.bfloat16).view(torch.int16), got[n].view(torch.int16))


def test_helper_keeps_an_own_classifier_and_the_fp32_rest():
    shape = SHAPES["tiny-qwen"]
    from kuiperllama_b200 import synth_weights
    w = synth_weights(shape, "cpu", 3)
    w["wcls"] = torch.randn(shape.vocab_size, shape.dim)
    b = bf16_weights(w)
    assert torch.equal(b["wcls"], w["wcls"].to(torch.bfloat16))
    for n in ("tok_emb", "attn_norm", "ffn_norm", "final_norm", "bq", "bk", "bv"):
        assert b[n] is w[n]
    w["wcls"] = None
    assert torch.equal(bf16_weights(w)["wcls"], w["tok_emb"].to(torch.bfloat16))
    assert w["wcls"] is None  # the fp32 dict is left as it was


def test_weight_bytes_per_token():
    t = SHAPES["tinyllama-1.1b"]
    f32, b16 = t.weight_bytes_per_token(), t.weight_bytes_per_token("bf16")
    d, h, L, kv, V = t.dim, t.hidden_dim, t.layer_num, t.kv_dim, t.vocab_size
    numel = L * (2 * d * d + 2 * kv * d + 3 * h * d) + V * d
    assert f32 - b16 == 2 * numel
    assert round(b16 / 1e9, 2) == 2.07 and round(f32 / 1e9, 2) == 4.14
    assert round(SHAPES["llama2-7b"].weight_bytes_per_token("bf16") / 1e9, 1) == 13.2
    with pytest.raises(ValueError):
        SHAPES["llama2-7b-int8"].weight_bytes_per_token("bf16")


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_decoder_desc_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text(f'#include <stddef.h>\n#include <stdio.h>\n#include "{HEADER_PATH}"\n'
                   'int main(void) { printf("%zu %zu %zu %d %d\\n", sizeof(kllm_decoder_desc), '
                   'offsetof(kllm_decoder_desc, kv_cache), offsetof(kllm_decoder_desc, weights), '
                   'KLLM_WEIGHTS_F32, KLLM_WEIGHTS_BF16); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.run(["cc", str(src), "-o", str(exe)], check=True)
    size, kv_off, w_off, f32, bf16 = map(int, subprocess.run([str(exe)], capture_output=True, text=True,
                                                              check=True).stdout.split())
    import ctypes
    assert (size, kv_off, w_off) == (ctypes.sizeof(DecoderDesc), DecoderDesc.kv_cache.offset,
                                     DecoderDesc.weights.offset)
    assert (f32, bf16) == (0, 1)
    assert DecoderDesc().weights == 0  # a zeroed struct: fp32

