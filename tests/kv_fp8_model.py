"""The fp8 KV cache's rule (kllm_decoder_desc::kv_cache = KLLM_KV_FP8) on top of the fp64 model of
tests/prefill_model.py, for tests/test_kv_fp8_model.py and tests/test_kv_fp8_gpu.py.

Rule: an element x of a K row (after RoPE) or a V row at layer l, KV head h is cached as the e4m3 code of
fp32(x * inv), inv = fp32(1 / s), round to nearest even and saturated to +-448; the code stands for fp32(value * s),
which is what the model attends over (and what kllm_decoder_read_kv returns).  The positions are the bf16 cache's
(tests/kv_bf16_model.py): "decode" attends over cached rows < p and the own row p unrounded, "prefill" over cached rows
only.  prefill_ref_fp8 is kv_bf16_model.prefill_ref_bf16 with a layer-counting kv_round.
"""
from __future__ import annotations

import numpy as np
import torch

from kv_bf16_model import prefill_ref_bf16

FP8_MAX = 448.0


def scaled(x, inv):
    """fp32(x * inv) of fp32 values x (the product of two fp32 values is exact in fp64, then rounded once)."""
    x = torch.as_tensor(x).to(torch.float32)
    return (x.double() * float(np.float32(inv))).to(torch.float32)


def e4m3_rne(y, trunc=False):
    """The e4m3 value of fp32 y: round to nearest even onto 3 mantissa bits (exponent floor -6, so the spacing below
    2^-6 is the subnormals' 2^-9), saturated to +-448; +-0 keep their sign; NaN stays NaN.  trunc: round toward zero
    instead (the tests' negative control).  Returns fp32 values, every one exactly an e4m3 value."""
    y = torch.as_tensor(y).to(torch.float32).double()
    a = y.abs()
    _, e = torch.frexp(a)  # a = m 2^e, m in [0.5, 1): spacing 2^(e - 4), at least 2^-9
    spacing = torch.pow(2.0, (torch.clamp(e, min=-5) - 4).double())
    q = a / spacing
    q = torch.trunc(q) if trunc else torch.round(q)  # torch.round: half to even
    v = torch.clamp(q * spacing, max=FP8_MAX)
    v = torch.where(torch.isnan(y), y, torch.copysign(v, y))
    return v.to(torch.float32)


def e4m3_codes(v):
    """The code bytes of e4m3 values v (exact: each converts without rounding)."""
    return torch.as_tensor(v).to(torch.float32).to(torch.float8_e4m3fn).view(torch.uint8)


def read_value(v, s):
    """fp32(v * s): a cached code's real value at scale s."""
    return scaled(v, s)


def kv_round_fp8(scales, trunc=False, ignore_scales=False):
    """A kv_round for prefill_ref_bf16 applying the fp8 rule with scales [2, L, kv_heads] (None: all 1).  It counts
    its calls: the attention of layer l rounds K then V, so call 2 l is layer l's K and 2 l + 1 its V.  Rows are
    [n, kv_heads, hs].  ignore_scales: encode at the scales but read the codes' values unscaled (a negative control)."""
    calls = [0]

    def kv_round(rows):
        c = calls[0]
        calls[0] += 1
        l, which = c // 2, c % 2
        rows = torch.as_tensor(rows)
        out = torch.empty(rows.shape, dtype=torch.float32, device=rows.device)
        for h in range(rows.shape[1]):
            s = 1.0 if scales is None else float(scales[which][l][h])
            inv = float(np.float32(1.0) / np.float32(s))
            v = e4m3_rne(scaled(rows[:, h], inv), trunc=trunc)
            out[:, h] = v if ignore_scales else read_value(v, s)
        return out

    return kv_round


def prefill_ref_fp8(weights, shape, tokens, start_pos, sin, cos, scales=None, rule="decode", trunc=False,
                    ignore_scales=False, kv_rows=None, **kw):
    """prefill_model.prefill_ref with the fp8 cache's rule at `scales` (see kv_round_fp8); kv_rows as in
    prefill_ref_bf16 (a decoder's read_kv rows, taken as given).  The rows returned are the model's own, unrounded."""
    return prefill_ref_bf16(weights, shape, tokens, start_pos, sin, cos, rule=rule,
                            kv_round=kv_round_fp8(scales, trunc, ignore_scales), kv_rows=kv_rows, **kw)


def fp8_round_rows(rows, scales, which):
    """The rule applied to whole cache rows [L, n, kv_dim] (a model's k or v) at scales[which] [L, kv_heads]:
    fp32(value(code) * s) per element."""
    rows = torch.as_tensor(rows).to(torch.float32)
    L, n, kvd = rows.shape
    kvh = scales.shape[-1] if scales is not None else None
    out = torch.empty_like(rows)
    for l in range(L):
        r = rows[l].reshape(n, kvh, kvd // kvh)
        for h in range(kvh):
            s = float(scales[which][l][h])
            inv = float(np.float32(1.0) / np.float32(s))
            out[l].view(n, kvh, -1)[:, h] = read_value(e4m3_rne(scaled(r[:, h], inv)), s)
    return out


def ulp_e4m3(v):
    """One e4m3 ulp at |v|: 2^(e - 3) for |v| in [2^e, 2^(e + 1)), 2^-9 below 2^-6.  The bounds take it at the larger
    of the two values compared: two elements on either side of a power of two are a step of the upper binade apart."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -6)))
    return torch.pow(2.0, e - 3)


def per_head(scales, which, L, kvh, hs, device):
    """The [L, 1, kv_dim] broadcast of scales[which] [L, kv_heads]."""
    s = torch.as_tensor(np.asarray(scales[which], np.float32), device=device).double()
    return s.repeat_interleave(hs, dim=1).reshape(L, 1, kvh * hs)
