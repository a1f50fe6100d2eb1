"""fp64 model of what the batched prompt prefill (csrc/prefill_gemm.cu, csrc/prefill.cu and the last position's
classifier in csrc/decoder.cu prefill()) and the decode step (csrc/megakernel.cu, both numerics modes) compute, for
the tests to hold the kernels against.  Row p of a causal forward over tokens 0 .. p is what a decode step at
position p computes, so one forward serves both.

The prefill multiplies on the tensor cores with both operands rounded to TF32 (cvt.rna: 10 explicit
mantissa bits, nearest, ties away from zero), accumulates in fp32 and stores every activation as fp32.  This
module does the same operations in float64, rounds the GEMM operands with the same rule, and rounds to fp32 at
every point the kernels store fp32.  A TF32 x TF32 product is exact in fp64 (11 + 11 significant bits), so
what is left between a correct kernel and this model is the order and rounding of fp32 accumulation and of
the fp32 element-wise arithmetic -- and the rare TF32 rounding decision that an fp32 difference of one unit
flips.  With `tf32=False` no operand is rounded to TF32: that is the plain fp32 model the CPU oracle
(oracle/kuiper_oracle.c) computes, which is how tests/test_prefill_model.py checks this module, and what the
decode step computes in its exact mode.

The decode step's fast mode (`numerics = fast`) rewrites the input vector of every int8 projection with group size
64 as 24-bit fixed point per 64-element group before the dot products (quantize_input_inplace,
accum_w8_dp4a); `fixed_point=True` replaces those inputs with the same fixed-point values (`fixed_point_value`, a
mirror of the kernel's fp32 arithmetic), so that what remains is again fp32 summation order.  Its attention
(flash-decoding) reorders the softmax sums only, which the exact softmax here stands for.

The forward is written from the operations, following the model's formulas (rmsnorm, q/k/v with the Qwen
bias, RoPE with interleaved (llama2) or half-split (qwen2) pairs, causal attention with grouped kv heads,
SwiGLU, residual adds), not from either implementation.  torch float64, on whatever device the inputs are.
"""
from __future__ import annotations

import numpy as np
import torch


def tf32_rna(t):
    """cvt.rna.tf32.f32 on fp32 values: add half a TF32 unit to the magnitude bits, (u + 0x1000) & ~0x1FFF,
    which rounds to nearest with ties away from zero and carries into the exponent (1.9999999 -> 2.0, the
    largest finite floats -> inf).  inf and NaN pass through; subnormals round on the same bit positions."""
    t = torch.as_tensor(t).to(torch.float32).contiguous()
    u = t.view(torch.int32)
    mag = u & 0x7FFFFFFF
    rounded = (u & -0x80000000) | ((mag + 0x1000) & ~0x1FFF)
    return torch.where(mag < 0x7F800000, rounded, u).view(torch.float32)


def f32(t):
    """fp64 -> the fp32 value the kernel stores, kept as fp64."""
    return t.to(torch.float32).to(torch.float64)


def dequant_w8(q, scales, group_size, tf32=True):
    """int8 weight [N, K] with one fp32 scale per `group_size` consecutive elements of the flattened matrix, as
    the GEMM's shared-memory tile holds it: fp32(scale * q), then rounded to TF32 (dequant_w8 in
    prefill_gemm.cu).  fp32 result."""
    q = torch.as_tensor(q)
    n, k = q.shape
    s = torch.as_tensor(scales).to(torch.float32).reshape(-1)[: n * k // group_size]
    w = s.repeat_interleave(group_size).reshape(n, k) * q.to(torch.float32)
    return tf32_rna(w) if tf32 else w


def gemm_operand(w, tf32=True):
    w = torch.as_tensor(w).to(torch.float32)
    return tf32_rna(w) if tf32 else w


def gemm_ref(x, w, tf32=True):
    """out[T, N] = x[T, K] . w[N, K]^T with both operands rounded to TF32 (unless tf32=False), multiplied and
    summed in fp64.  fp64 result, not rounded."""
    return gemm_operand(x, tf32).to(torch.float64) @ gemm_operand(w, tf32).to(torch.float64).t()


def gemm_abs_ref(x, w, tf32=True):
    """sum_k |x~[t, k] w~[n, k]|: the scale of the fp32 accumulation error of out[t, n]."""
    return gemm_operand(x, tf32).to(torch.float64).abs() @ gemm_operand(w, tf32).to(torch.float64).abs().t()


FP_ONE = 4194304.0  # 2^22: the fixed point's full scale, q = +-2^22 at the group maximum


def balanced_digits(q):
    """q (integers, |q| <= 2^22) -> (a2, a1, a0) with q = 65536 a2 + 256 a1 + a0 and a0, a1 in [-128, 127]: the
    kernel's balanced base-256 split (quantize_input_inplace).  numpy or torch integer arrays."""
    a0 = ((q + 128) & 255) - 128
    q1 = (q - a0) >> 8
    a1 = ((q1 + 128) & 255) - 128
    return (q1 - a1) >> 8, a1, a0


def fixed_point_parts(x):
    """The fast mode's fixed point of x [..., M] (M % 64 == 0), in the kernel's fp32 arithmetic, per 64-element
    group: gmax = max|x|, step = fp32(gmax * 2^-22), inv = fp32(2^22 / gmax) (0 when gmax is 0), q = x * inv
    rounded to fp32, then to the nearest integer (ties to even, __float2int_rn).  Returns (step [..., M / 64, 1],
    q [..., M / 64, 64]) as fp32 tensors."""
    x = torch.as_tensor(x).to(torch.float32)
    xg = x.reshape(*x.shape[:-1], x.shape[-1] // 64, 64)
    gmax = xg.abs().amax(dim=-1, keepdim=True)
    step = gmax * np.float32(1.0 / FP_ONE)
    inv = torch.where(gmax > 0, np.float32(FP_ONE) / gmax, torch.zeros_like(gmax))
    return step, torch.round(xg * inv)


def fixed_point_value(x):
    """step * q for every element of x [..., M]: the value the fast mode's int8 dot products see, exact in fp64
    (not an fp32 value: 24-bit step times 23-bit q)."""
    step, q = fixed_point_parts(x)
    return (step.to(torch.float64) * q.to(torch.float64)).reshape(x.shape)


def flavour_eps(flavour):
    return 1e-6 if flavour == "qwen2" else 1e-5


def _t(a, device):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.array(a, copy=True))
    return a.to(device)


def _rmsnorm(x, w, eps):
    eps = float(np.float32(eps))
    return f32(x * torch.rsqrt((x * x).mean(dim=-1, keepdim=True) + eps) * w.to(torch.float64))


def _rope(x, sin, cos, pos, flavour):
    """x [n, heads, hs] fp64; pair (i0, i1) of rotation j uses the table at column 2j of row pos."""
    hs = x.shape[-1]
    half = hs // 2
    j = torch.arange(half, device=x.device)
    i0, i1 = (2 * j, 2 * j + 1) if flavour == "llama2" else (j, j + half)
    s = sin[pos][:, 2 * j].to(torch.float64)[:, None, :]
    c = cos[pos][:, 2 * j].to(torch.float64)[:, None, :]
    a, b = x[..., i0], x[..., i1]
    out = torch.empty_like(x)
    out[..., i0] = f32(a * c - b * s)
    out[..., i1] = f32(a * s + b * c)
    return out


def _attention(q, k_all, v_all, start_pos, kv_mul, max_bytes=1 << 28):
    """Causal attention of the n query rows at positions start_pos .. start_pos + n - 1 over cache rows
    0 .. pos (the query's own position included).  q [n, heads, hs], k_all / v_all [P, kv_heads, hs], all fp64.
    Chunked by query rows so that the scores of 12k+ positions fit in `max_bytes`."""
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
        o = torch.softmax(s, dim=-1) @ vt[:, :P]  # [kvh, rows * kv_mul, hs]
        out[t0:t1] = o.reshape(kvh, t1 - t0, kv_mul, hs).permute(1, 0, 2, 3).reshape(t1 - t0, heads, hs)
    return f32(out)


def layer_ops(weights, shape, dev, tf32, fixed_point):
    """(proj, bias), the projections of one layer as prefill_ref computes them: proj(x, name, l) is
    fp32(operand(x) . W^T) with the layer's matrix widened (int8: dequantised) when it is used, operand(x) x rounded to
    TF32 (tf32) or the fast mode's fixed point (fixed_point, int8 group size 64); bias(y, name, l) adds the Qwen bias
    where the weights have one."""
    g = shape.group_size

    def weight(name, l):
        w = weights[name][l]
        if g:
            return dequant_w8(_t(w, dev), _t(weights["s" + name[1:]][l], dev), g, tf32)
        return gemm_operand(_t(w, dev), tf32)

    def operand(x):
        if fixed_point and g == 64 and x.shape[-1] % 64 == 0:
            return fixed_point_value(x)
        return gemm_operand(x.to(torch.float32), tf32).to(torch.float64)

    def proj(x, name, l):
        return f32(operand(x) @ weight(name, l).to(torch.float64).t())

    def bias(y, name, l):
        b = weights.get(name)
        return y if b is None else f32(y + _t(b[l], dev).to(torch.float64))

    return proj, bias


def classify(weights, shape, x, dev, fixed_point):
    """The final RMSNorm and the classifier of the rows x [n, dim]: fp64 logits [n, vocab] of the fp32 classifier (no
    TF32: it is the decode path's GEMV), its input in the fast mode's fixed point with fixed_point."""
    g = shape.group_size
    xl = _rmsnorm(x, _t(weights["final_norm"], dev), flavour_eps(shape.flavour))
    wcls = weights.get("wcls")
    if wcls is None:
        wcls = weights["tok_emb"]
    if g:
        wc = dequant_w8(_t(wcls, dev), _t(weights["scls"], dev), g, tf32=False)
    else:
        wc = _t(wcls, dev)
    if fixed_point and g == 64 and shape.dim % 64 == 0:
        xl = fixed_point_value(xl)
    return xl @ wc.to(torch.float64).t()


def prefill_ref(weights, shape, tokens, start_pos, sin, cos, kv_in=None, tf32=True, device=None, logits_at=(),
                fixed_point=False):
    """The forward of prefill_block over `tokens` at positions start_pos .. start_pos + n - 1, then the last
    position's final RMSNorm and classifier (and those of the rows listed in `logits_at`: what a prefill of
    tokens[:i + 1] would leave, since no row depends on a later one).

    weights   dict as synth_weights / read_checkpoint give it (torch or numpy; int8 with s* scales; bq/bk/bv for
              the Qwen bias; wcls None = the embedding is the classifier)
    sin, cos  the [seq_len, head_size] tables the kernels read (on the GPU: what kllm_sincos_init wrote)
    kv_in     (k, v) [L, >= start_pos, kv_dim]: the cache rows before start_pos
    fixed_point  the decode step's fast mode: the input of every int8 projection with group size 64 and an input
              length divisible by 64 (q/k/v, Wo, W1/W3, W2 and the classifier) becomes fixed_point_value(x).
              Needs tf32=False.
    Returns dict: k, v [L, n, kv_dim] (the cache rows written, after RoPE for k), logits [vocab] (fp64 of the
    fp32 classifier: no TF32 there, it is the decode path's GEMV), next (first maximum) and logits_at
    {row: logits}."""
    s = shape
    dev = device or (weights["tok_emb"].device if isinstance(weights["tok_emb"], torch.Tensor) else "cpu")
    L, hs, heads, kvh = s.layer_num, s.head_size, s.head_num, s.kv_head_num
    n = len(tokens)
    eps = flavour_eps(s.flavour)
    assert not (fixed_point and tf32), "the fixed point is the decode step's; the prefill's GEMMs are TF32"
    sin, cos = _t(sin, dev), _t(cos, dev)
    pos = torch.arange(start_pos, start_pos + n, device=dev)
    tok = torch.as_tensor(np.asarray(tokens, dtype=np.int64), device=dev)

    proj, bias = layer_ops(weights, s, dev, tf32, fixed_point)

    x = _t(weights["tok_emb"], dev)[tok].to(torch.float64)
    ks, vs = [], []
    for l in range(L):
        xn = _rmsnorm(x, _t(weights["attn_norm"][l], dev), eps)
        q = bias(proj(xn, "wq", l), "bq", l).reshape(n, heads, hs)
        k = bias(proj(xn, "wk", l), "bk", l).reshape(n, kvh, hs)
        v = bias(proj(xn, "wv", l), "bv", l).reshape(n, kvh, hs)
        q = _rope(q, sin, cos, pos, s.flavour)
        k = _rope(k, sin, cos, pos, s.flavour)
        ks.append(k.reshape(n, -1))
        vs.append(v.reshape(n, -1))
        if start_pos > 0:
            k_prev = _t(kv_in[0][l][:start_pos], dev).to(torch.float64).reshape(start_pos, kvh, hs)
            v_prev = _t(kv_in[1][l][:start_pos], dev).to(torch.float64).reshape(start_pos, kvh, hs)
            k, v = torch.cat([k_prev, k]), torch.cat([v_prev, v])
        att = _attention(q, k, v, start_pos, heads // kvh).reshape(n, -1)
        x = f32(x + proj(att, "wo", l))
        xn = _rmsnorm(x, _t(weights["ffn_norm"][l], dev), eps)
        h1, h3 = proj(xn, "w1", l), proj(xn, "w3", l)
        h = f32(h1 * torch.sigmoid(h1) * h3)
        x = f32(x + proj(h, "w2", l))
    rows = sorted({i % n for i in logits_at} | {n - 1})
    logits = dict(zip(rows, classify(weights, s, x[rows], dev, fixed_point)))
    last = logits[n - 1]
    return {"k": torch.stack(ks), "v": torch.stack(vs), "logits": last, "next": int(torch.argmax(last)),
            "logits_at": logits}
