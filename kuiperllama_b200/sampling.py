"""numpy mirror of the sampling rule of ``csrc/sampling.cuh`` (the one other place the rule is written
down).  The tests compare every device path against it; DESIGN.md "Sampling" gives the reasons.
"""
from __future__ import annotations

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 on arrays: ctr is [..., 4] uint32, key a pair of ints; returns [..., 4] uint32."""
    c = np.asarray(ctr, dtype=np.uint64).copy()
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0 = _M0 * c[..., 0]
        p1 = _M1 * c[..., 2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c = np.stack([hi1 ^ c[..., 1] ^ np.uint64(k0), lo1, hi0 ^ c[..., 3] ^ np.uint64(k1), lo0], axis=-1)
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return c.astype(np.uint32)


def gumbel_noise(n: int, seed: int, pos: int) -> np.ndarray:
    """g_i, i < n, for (seed, pos): word i & 3 of the Philox block at counter (i >> 2, pos, 0, 0)."""
    blocks = (n + 3) // 4
    ctr = np.zeros((blocks, 4), np.uint64)
    ctr[:, 0] = np.arange(blocks)
    ctr[:, 1] = pos
    return gumbel(philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).reshape(-1)[:n])


def uniform(x) -> np.ndarray:
    """u of Philox words x: ((x >> 8) + 0.5) * 2^-24 rounded toward zero to fp32, so that u < 1 (k + 0.5
    needs a 25th bit once k = x >> 8 >= 2^23; rounding to nearest would give u = 1 for the largest k)."""
    k = (np.asarray(x, np.uint32) >> np.uint32(8)).astype(np.int64)
    return (np.where(k >= 1 << 23, k, k + 0.5) * 2.0 ** -24).astype(np.float32)


def gumbel(x) -> np.ndarray:
    """g = -log(-log(u)) of Philox words x, in fp32."""
    return -np.log(-np.log(uniform(x)))


def scores(logits, temperature: float, top_k: int, seed: int, pos: int):
    """s_i + g_i for the kept i, -inf for the others (temperature > 0)."""
    s = np.asarray(logits, np.float32) / np.float32(temperature)
    n = s.shape[0]
    v = s + gumbel_noise(n, seed, pos)
    if 0 < top_k < n:
        tau = np.partition(s, n - top_k)[n - top_k]
        v = np.where(s >= tau, v, np.float32(-np.inf))
    return v


def sample(logits, temperature: float, top_k: int, seed: int, pos: int) -> int:
    """The id the rule draws from `logits` at position `pos` (greedy for temperature 0)."""
    if temperature == 0:
        return int(np.argmax(np.asarray(logits, np.float32)))
    return int(np.argmax(scores(logits, temperature, top_k, seed, pos)))


def margin(logits, temperature: float, top_k: int, seed: int, pos: int) -> float:
    """Relative gap between the two best perturbed scores: below ~1e-5 a last-ulp difference of the
    device logf may change the id."""
    if temperature == 0:
        v = np.asarray(logits, np.float32)
    else:
        v = scores(logits, temperature, top_k, seed, pos)
    top2 = np.partition(v, v.shape[0] - 2)[-2:]
    if not np.isfinite(top2).all():
        return float("inf")
    return float((top2[1] - top2[0]) / max(abs(float(top2[1])), 1.0))
