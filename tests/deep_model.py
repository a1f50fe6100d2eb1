"""A layer-streamed, position-sampled fp64 model of the decoder, for holding full-size models (a 7B model widened to
fp64 is about 52 GB) to the arithmetic of tests/prefill_model.py at full depth and full context.

Given the weights, a set of positions P, the id fed at each and the decoder's own cache rows (kllm_decoder_read_kv's,
one layer at a time), `sampled_ref` runs only the rows of P through the layers.  Each layer's matrices are widened to
fp64 (int8 ones dequantised) one at a time and dropped after use.  Row p attends over the decoder's cached rows of that
layer:
  - "decode": rows [0, p) as cached, and its own row p unrounded (what a decode step does, whatever the cache's element:
    the fp32 cache stores that row unrounded, and the bf16 and fp8 caches' decode rule attends over it before rounding;
    tests/kv_bf16_model.py, tests/kv_fp8_model.py);
  - "prefill": rows [0, p] as cached, its own included (the batched prefill attends over what it cached).
Because every row attends over the rows the decoder actually cached, the error does not build up along the positions:
a check at position 4000 is as tight as one at position 40; only the depth adds up.

The arithmetic is prefill_model's: its RMSNorm, RoPE, projections (layer_ops: the prefill's TF32 operands, the fast
mode's fixed point, int8 dequantisation) and classifier (classify); only the attention over sampled rows is this
module's.  tests/test_deep_model.py pins it to prefill_model.prefill_ref on small shapes.
"""
from __future__ import annotations

import numpy as np
import torch

from prefill_model import _rmsnorm, _rope, _t, classify, f32, flavour_eps, layer_ops


def sampled_ref(weights, shape, positions, tokens, sin, cos, kv_rows, rule="decode", tf32=False, fixed_point=False,
                device=None):
    """The forward of the rows at `positions` (sorted, distinct) fed `tokens` (one id each).

    kv_rows   callable l -> (k, v) [> max(positions), kv_dim]: the decoder's cache rows of layer l, as read_kv returns
              them (torch or numpy); asked for once per layer, in order
    rule      "decode" or "prefill" (see the module's docstring)
    tf32, fixed_point  as prefill_ref: tf32 for the batched prefill's rows, fixed_point for the fast mode's decode rows
    Returns dict: k, v [L, n, kv_dim] (the rows the model computes at P, after RoPE for k; unrounded), logits {p: [vocab]}
    and next {p: first maximum}."""
    assert rule in ("decode", "prefill"), rule
    assert not (fixed_point and tf32), "the fixed point is the decode step's; the prefill's GEMMs are TF32"
    s = shape
    dev = device or (weights["tok_emb"].device if isinstance(weights["tok_emb"], torch.Tensor) else "cpu")
    L, hs, heads, kvh = s.layer_num, s.head_size, s.head_num, s.kv_head_num
    kv_mul = heads // kvh
    positions = [int(p) for p in positions]
    assert positions == sorted(set(positions)), positions
    n = len(positions)
    eps = flavour_eps(s.flavour)
    sin, cos = _t(sin, dev), _t(cos, dev)
    pos = torch.as_tensor(positions, device=dev)
    tok = torch.as_tensor(np.asarray(tokens, dtype=np.int64), device=dev)

    proj, bias = layer_ops(weights, s, dev, tf32, fixed_point)  # one matrix widened at a time

    x = _t(weights["tok_emb"], dev)[tok].to(torch.float64)
    ks, vs = [], []
    scale = 1.0 / np.sqrt(hs)
    for l in range(L):
        xn = _rmsnorm(x, _t(weights["attn_norm"][l], dev), eps)
        q = bias(proj(xn, "wq", l), "bq", l).reshape(n, heads, hs)
        k = bias(proj(xn, "wk", l), "bk", l).reshape(n, kvh, hs)
        v = bias(proj(xn, "wv", l), "bv", l).reshape(n, kvh, hs)
        q = _rope(q, sin, cos, pos, s.flavour)
        k = _rope(k, sin, cos, pos, s.flavour)
        ks.append(k.reshape(n, -1))
        vs.append(v.reshape(n, -1))
        kc, vc = kv_rows(l)
        top = positions[-1] + 1
        kc = _t(torch.as_tensor(kc[:top]), dev).to(torch.float64).reshape(top, kvh, hs).permute(1, 0, 2)  # [kvh, P, hs]
        vc = _t(torch.as_tensor(vc[:top]), dev).to(torch.float64).reshape(top, kvh, hs).permute(1, 0, 2)
        att = torch.empty(n, heads, hs, dtype=torch.float64, device=dev)
        for i, p in enumerate(positions):
            qg = q[i].reshape(kvh, kv_mul, hs)
            if rule == "decode":  # cached rows [0, p), then the own row
                K = torch.cat([kc[:, :p], k[i][:, None]], dim=1)
                V = torch.cat([vc[:, :p], v[i][:, None]], dim=1)
            else:
                K, V = kc[:, :p + 1], vc[:, :p + 1]
            sc = (qg @ K.transpose(1, 2)) * scale  # [kvh, kv_mul, p + 1]
            att[i] = (torch.softmax(sc, dim=-1) @ V).reshape(heads, hs)
        del kc, vc
        x = f32(x + proj(f32(att).reshape(n, -1), "wo", l))
        xn = _rmsnorm(x, _t(weights["ffn_norm"][l], dev), eps)
        h1, h3 = proj(xn, "w1", l), proj(xn, "w3", l)
        h = f32(h1 * torch.sigmoid(h1) * h3)
        del h1, h3
        x = f32(x + proj(h, "w2", l))
    logits = classify(weights, s, x, dev, fixed_point)
    return {"k": torch.stack(ks), "v": torch.stack(vs), "logits": dict(zip(positions, logits)),
            "next": {p: int(torch.argmax(lg)) for p, lg in zip(positions, logits)}}
