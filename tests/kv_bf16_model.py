"""The bf16 KV cache's rounding rule (kllm_decoder_desc::kv_cache = KLLM_KV_BF16) on top of the fp64 model of
tests/prefill_model.py, for tests/test_kv_bf16_model.py and tests/test_kv_bf16_gpu.py.

Rule: every K row (after RoPE) and V row is cached as bf16 (round to nearest even).  A decode step at position p
attends over the cached rows < p and over its own row p unrounded ("decode"); the batched prefill attends over cached
rows only, its own included ("prefill"); "all" is the decode step with row p rounded too (a negative control).

prefill_ref_bf16 runs prefill_model.prefill_ref unchanged and replaces only its attention, for the duration of the
call, by one that applies the rule: the forward, the rows it returns and the logits are prefill_ref's.
"""
from __future__ import annotations

import numpy as np
import torch

import prefill_model
from prefill_model import f32


def bf16_rne(t):
    """fp32 -> bf16 -> fp32 by round to nearest, ties to even (__float2bfloat16_rn, the bf16 KV cache's rounding):
    add 0x7FFF plus the lowest kept bit to the bits, clear the low 16.  Carries into the exponent (to inf past the
    largest bf16); subnormals round on the same bit positions; +-0 keep their sign; NaN passes through."""
    t = torch.as_tensor(t).to(torch.float32).contiguous()
    u = t.view(torch.int32)
    rounded = (u + 0x7FFF + ((u >> 16) & 1)) & -0x10000
    return torch.where((u & 0x7FFFFFFF) <= 0x7F800000, rounded, u).view(torch.float32)


def bf16_trunc(t):
    """fp32 -> bf16 by truncation: the rounding a bf16 cache must NOT use (the tests' negative control)."""
    t = torch.as_tensor(t).to(torch.float32).contiguous()
    return (t.view(torch.int32) & -0x10000).view(torch.float32)


def attention_own_row(q, k_all, v_all, start_pos, kv_mul, k_own, v_own, max_bytes=1 << 28):
    """prefill_model's causal attention of the n query rows at positions start_pos .. start_pos + n - 1 over rows
    0 .. pos of k_all / v_all [P, kv_heads, hs], except that each query's OWN position takes k_own / v_own
    [n, kv_heads, hs] (the decode rule: earlier rows as cached, the current one unrounded).  fp64 in, fp32 out."""
    n, heads, hs = q.shape
    kvh = heads // kv_mul
    out = torch.empty_like(q)
    kt = k_all.permute(1, 2, 0)  # [kvh, hs, P]
    vt = v_all.permute(1, 0, 2)  # [kvh, P, hs]
    rows = max(1, int(max_bytes // (8 * heads * (start_pos + n))))
    scale = 1.0 / np.sqrt(hs)
    for t0 in range(0, n, rows):
        t1 = min(n, t0 + rows)
        P = start_pos + t1
        qc = q[t0:t1].reshape(t1 - t0, kvh, kv_mul, hs).permute(1, 0, 2, 3).reshape(kvh, -1, hs)
        s = (qc @ kt[:, :, :P]) * scale  # [kvh, rows * kv_mul, P]
        pos = torch.arange(start_pos + t0, start_pos + t1, device=q.device).repeat_interleave(kv_mul)
        s = s.masked_fill(torch.arange(P, device=q.device)[None, None, :] > pos[None, :, None], float("-inf"))
        kc = k_own[t0:t1].permute(1, 0, 2).repeat_interleave(kv_mul, dim=1)  # [kvh, rows * kv_mul, hs]
        vc = v_own[t0:t1].permute(1, 0, 2).repeat_interleave(kv_mul, dim=1)
        col = pos[None, :, None].expand(kvh, -1, 1)
        s = s.scatter(-1, col, (qc * kc).sum(-1, keepdim=True) * scale)  # the own row's score
        p = torch.softmax(s, dim=-1)
        o = p @ vt[:, :P] + p.gather(-1, col) * (vc - vt.gather(1, col.expand(-1, -1, hs)))  # ... and its value
        out[t0:t1] = o.reshape(kvh, t1 - t0, kv_mul, hs).permute(1, 0, 2, 3).reshape(t1 - t0, heads, hs)
    return f32(out)


def prefill_ref_bf16(weights, shape, tokens, start_pos, sin, cos, rule="decode", kv_round=bf16_rne, kv_rows=None,
                     **kw):
    """prefill_model.prefill_ref (same arguments in **kw: kv_in, tf32, logits_at, fixed_point, ...) with the bf16
    cache's rule: the rows of these positions are cached as kv_round(row), or, with kv_rows ((k, v) [L, >= n,
    kv_dim], a decoder's read_kv), taken as given -- so that each position attends over the rows the decoder
    actually cached.  kv_in rows are taken as given (a bf16 decoder's read_kv rows are bf16 already).  The rows
    returned are the model's own, unrounded."""
    assert rule in ("decode", "prefill", "all"), rule
    n = len(tokens)
    layer = [0]

    def attention(q, k_all, v_all, sp, kv_mul):
        l = layer[0]
        layer[0] += 1
        kvh, hs = k_all.shape[1], k_all.shape[2]
        k_own, v_own = k_all[sp:], v_all[sp:]
        if kv_rows is None:
            k_c, v_c = kv_round(k_own).to(torch.float64), kv_round(v_own).to(torch.float64)
        else:
            k_c = kv_rows[0][l][:n].to(q.device, torch.float64).reshape(n, kvh, hs)
            v_c = kv_rows[1][l][:n].to(q.device, torch.float64).reshape(n, kvh, hs)
        k_c, v_c = torch.cat([k_all[:sp], k_c]), torch.cat([v_all[:sp], v_c])
        if rule == "decode":
            return attention_own_row(q, k_c, v_c, sp, kv_mul, k_own, v_own)
        return plain(q, k_c, v_c, sp, kv_mul)

    plain = prefill_model._attention
    prefill_model._attention = attention
    try:
        return prefill_model.prefill_ref(weights, shape, tokens, start_pos, sin, cos, **kw)
    finally:
        prefill_model._attention = plain
