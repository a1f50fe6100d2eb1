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


def history_window(history, pos: int, last_n: int = 0) -> np.ndarray:
    """Step 0's H(pos): the entries of `history` (the id fed at each position, < 0 for none) at positions
    [lo, pos], lo = 0 for last_n == 0 else max(0, pos - last_n + 1)."""
    lo = 0 if last_n == 0 else max(0, pos - last_n + 1)
    return np.asarray(history, np.int64)[lo:pos + 1]


def penalize(logits, ids, penalty: float) -> np.ndarray:
    """Step 0b: l_i * theta for negative l_i, else l_i / theta, for every i in `ids` (ids < 0 or >= len(logits)
    ignored, duplicates penalised once), theta = fp32(penalty); the other logits unchanged."""
    out = np.array(logits, np.float32, copy=True)
    ids = np.asarray(ids, np.int64)
    ids = np.unique(ids[(ids >= 0) & (ids < out.shape[0])])
    theta = np.float32(penalty)
    l = out[ids]
    with np.errstate(over="ignore"):  # both branches are evaluated; an overflow to inf is the fp32 result
        out[ids] = np.where(l < 0, l * theta, l / theta)
    return out


def bias_table(mapping, n: int):
    """Step 0a's dense table [n] fp32 of an {id: bias} map (unset entries 0), or None for an empty map: then the
    step is skipped, which keeps the sign of a -0.0 logit.  Each entry is 0 + b, as HF builds its bias (a -0.0
    bias is +0.0)."""
    if not mapping:
        return None
    table = np.zeros(n, np.float32)
    for i, b in mapping.items():
        table[int(i)] += np.float32(b)
    return table


def apply_bias(logits, table) -> np.ndarray:
    """Step 0a: l_i + b_i for every i (one fp32 addition), or the logits unchanged when `table` is None."""
    out = np.array(logits, np.float32, copy=True)
    return out if table is None else out + np.asarray(table, np.float32)


def count_window(history, pos: int, from_pos: int) -> np.ndarray:
    """Steps 0c/0d's C(pos): the entries of `history` at positions [from_pos, pos] (empty for from_pos > pos)."""
    return np.asarray(history, np.int64)[max(0, from_pos):pos + 1]


def frequency_presence(logits, ids, frequency: float, presence: float) -> np.ndarray:
    """Steps 0c and 0d: for every i with c_i > 0 occurrences in `ids` (ids < 0 or >= len(logits) ignored),
    l_i - fp32(frequency) * fp32(c_i), then - fp32(presence), each one fp32 operation; a zero alpha skips its
    line.  The other logits unchanged."""
    out = np.array(logits, np.float32, copy=True)
    ids = np.asarray(ids, np.int64)
    ids = ids[(ids >= 0) & (ids < out.shape[0])]
    if ids.size == 0:
        return out
    counted, c = np.unique(ids, return_counts=True)
    f, p = np.float32(frequency), np.float32(presence)
    l = out[counted]
    with np.errstate(over="ignore"):
        if f != 0:
            l = l - f * c.astype(np.float32)
        if p != 0:
            l = l - p
    out[counted] = l
    return out


def penalties(logits, *, bias=None, rep_ids=(), penalty: float = 1.0, count_ids=(), frequency: float = 0.0,
              presence: float = 0.0) -> np.ndarray:
    """The whole of step 0 in its order: 0a bias (`bias` a dense table or None), 0b the repetition penalty over
    `rep_ids`, 0c frequency and 0d presence over the multiset `count_ids`."""
    out = apply_bias(logits, bias)
    if np.float32(penalty) != 1:
        out = penalize(out, rep_ids, penalty)
    return frequency_presence(out, count_ids, frequency, presence)


NUCLEUS_EPS = 1e-6
"""np.exp and the device expf may differ in the last ulps of each weight, which moves A and Z by well under
this much of Z: a nucleus comparison closer than that may go either way on the device."""


def top_p_active(temperature: float, top_p: float) -> bool:
    """Step 3b runs for T > 0 and 0 < top_p < 1 (top_p as the device's fp32)."""
    p = np.float32(top_p)
    return temperature > 0 and bool(0 < p < 1)


def nucleus_masses(s) -> np.ndarray:
    """q_i = floor(w_i * 2^32), w_i = exp(s_i - max s) in fp32, of the kept scores s (int64, exact)."""
    s = np.asarray(s, np.float32)
    w = np.exp(s - s.max())
    return np.floor(w.astype(np.float64) * 2.0 ** 32).astype(np.int64)


def _nucleus(s, top_p: float):
    """Over the kept scores s: the distinct values u (ascending), the mass strictly above each (A), Z, p24
    and J, the index in u of the smallest kept value."""
    u, inv = np.unique(np.asarray(s, np.float32), return_inverse=True)
    mass = np.zeros(u.shape[0], np.int64)
    np.add.at(mass, inv, nucleus_masses(s))
    above = np.concatenate([np.cumsum(mass[::-1])[::-1][1:], np.zeros(1, np.int64)])
    z = int(mass.sum())
    p24 = max(1, int(np.rint(np.float64(np.float32(top_p)) * 2.0 ** 24)))
    need = -(-p24 * z // 2 ** 24)  # A * 2^24 < p24 * Z  <=>  A < ceil(p24 * Z / 2^24), A an integer
    j = int(np.argmax(above < need))  # `above` falls as u grows; the largest value has A = 0 < need
    return u, above, z, p24, j


def nucleus_threshold(s, top_p: float) -> np.float32:
    """tau_p of step 3b over the kept scores s: keep s_i >= tau_p."""
    u, _, _, _, j = _nucleus(s, top_p)
    return u[j]


def _keep(s, top_k: int, top_p: float, shift: int = 0):
    """The kept set of steps 3 and 3b (shift moves tau_p by that many distinct values: the margin's what-if)."""
    n = s.shape[0]
    keep = np.ones(n, bool)
    if 0 < top_k < n:
        keep = s >= np.partition(s, n - top_k)[n - top_k]
    if top_p_active(1.0, top_p):
        u, _, _, _, j = _nucleus(s[keep], top_p)
        keep &= s >= u[min(max(j + shift, 0), u.shape[0] - 1)]
    return keep


def scores(logits, temperature: float, top_k: int, seed: int, pos: int, top_p: float = 1.0, _shift: int = 0):
    """s_i + g_i for the kept i, -inf for the others (temperature > 0)."""
    s = np.asarray(logits, np.float32) / np.float32(temperature)
    n = s.shape[0]
    v = s + gumbel_noise(n, seed, pos)
    if 0 < top_k < n or top_p_active(temperature, top_p):
        v = np.where(_keep(s, top_k, top_p, _shift), v, np.float32(-np.inf))
    return v


def sample(logits, temperature: float, top_k: int, seed: int, pos: int, top_p: float = 1.0) -> int:
    """The id the rule draws from `logits` at position `pos` (greedy for temperature 0)."""
    if temperature == 0:
        return int(np.argmax(np.asarray(logits, np.float32)))
    return int(np.argmax(scores(logits, temperature, top_k, seed, pos, top_p)))


def nucleus_size(logits, temperature: float, top_k: int, top_p: float) -> int:
    """How many tokens steps 3 and 3b keep (temperature > 0)."""
    s = np.asarray(logits, np.float32) / np.float32(temperature)
    return int(_keep(s, top_k, top_p if top_p_active(temperature, top_p) else 1.0).sum())


def nucleus_margin(logits, temperature: float, top_k: int, top_p: float) -> float:
    """How close step 3b's decisive comparisons (A * 2^24 against p24 * Z at the smallest kept value and the
    largest dropped one) are, relative to Z * 2^24; inf when top-p is off.  Below NUCLEUS_EPS the device may
    keep one value more or one less."""
    if not top_p_active(temperature, top_p):
        return float("inf")
    s = np.asarray(logits, np.float32) / np.float32(temperature)
    n = s.shape[0]
    kept = s[s >= np.partition(s, n - top_k)[n - top_k]] if 0 < top_k < n else s
    _, above, z, p24, j = _nucleus(kept, top_p)
    gaps = [abs(int(above[i]) * 2 ** 24 - p24 * z) for i in (j - 1, j) if i >= 0]
    return min(gaps) / (z * 2.0 ** 24)


MAX_TOP_LOGPROBS = 20


def top_n(logits, n: int) -> np.ndarray:
    """The n largest logits' ids in descending order, lowest index on ties (-1 pads past the vector's length)."""
    v = np.asarray(logits, np.float32)
    order = np.lexsort((np.arange(v.shape[0]), -v.astype(np.float64)))[:n]
    return np.concatenate([order, -np.ones(max(0, n - v.shape[0]), np.int64)]).astype(np.int64)


def warp_parts(n: int, w: int = 32):
    """The partition of the one-block kernels: w contiguous ranges [j n / w, (j + 1) n / w)."""
    return [(j * n // w, (j + 1) * n // w) for j in range(w)]


def logprobs(logits, ids, top_n_: int = 0, parts=None):
    """The logprob rule of csrc/sampling.cuh (DESIGN.md 5.8) over raw fp32 logits: (lp of each of `ids`, top-N ids,
    top-N lp).  parts=None: exact fp64 log_softmax.  Otherwise L1-L3 emulated in fp32 over the given partition
    (a list of (lo, hi) ranges), each part summed in increasing index order."""
    l = np.asarray(logits, np.float32)
    ids = np.asarray(ids, np.int64)
    top = top_n(l, top_n_)
    if parts is None:
        l64 = l.astype(np.float64)
        m = l64.max()
        lse = m + np.log(np.exp(l64 - m).sum())
        lp = lambda i: l64[i] - lse  # noqa: E731
    else:
        f = np.float32
        ms, ss = [], []
        for lo, hi in parts:
            if hi <= lo:
                ms.append(f(-np.inf)), ss.append(f(0))
                continue
            seg = l[lo:hi]
            mc = seg.max()
            # np.add.accumulate adds in order, one fp32 rounding per term (np.sum would add pairwise)
            ms.append(mc), ss.append(np.add.accumulate(np.exp(seg - mc).astype(np.float32), dtype=np.float32)[-1])
        m = max(ms)
        S = f(0)
        for mc, sc in zip(ms, ss):
            if sc > 0:
                S = f(S + f(sc * np.exp(f(mc - m))))
        lse_off = np.log(S).astype(np.float32)
        lp = lambda i: ((l[i] - m).astype(np.float32) - lse_off).astype(np.float32)  # noqa: E731
    lp_ids = np.array([lp(i) if 0 <= i < l.shape[0] else np.nan for i in ids], np.float64)
    lp_top = np.array([lp(i) if i >= 0 else -np.inf for i in top], np.float64)
    return lp_ids, top, lp_top


def logprob_bound(lp, chain: int, V: int) -> np.ndarray:
    """|lp - lp_fp64| <= (k + 10) u + 5 u log V + 2 u |lp|, u = 2^-24, for a computation of S whose longest chain of
    dependent fp32 additions is k (DESIGN.md 5.8 derives it)."""
    u = 2.0 ** -24
    return (chain + 10) * u + 5 * u * np.log(V) + 2 * u * np.abs(np.asarray(lp, np.float64))


def chain_of_parts(parts) -> int:
    """k of the emulation: a part summed in order, then the parts folded in order."""
    return max(hi - lo for lo, hi in parts) + len(parts)


def chain_persistent(V: int, grid: int, threads: int = 256) -> int:
    """k of the persistent engine: a thread's strided rows, the warp butterfly, the warps in order, the CTAs in order."""
    rows = -(-V // grid)
    return -(-rows // threads) + 5 + threads // 32 + grid


def chain_one_block(V: int) -> int:
    """k of the one-block kernels (graph engine, kllm_logprobs_f32): a lane's strided share of its warp's range, the
    butterfly, the 32 warps in order."""
    return -(-(-(-V // 32)) // 32) + 5 + 32


def margin(logits, temperature: float, top_k: int, seed: int, pos: int, top_p: float = 1.0) -> float:
    """Relative gap between the two best perturbed scores: below ~1e-5 a last-ulp difference of the
    device logf may change the id.  With top-p, 0 also when a nucleus comparison is within NUCLEUS_EPS
    (nucleus_margin) and keeping one value more or one less would change the id."""
    if temperature == 0:
        v = np.asarray(logits, np.float32)
    else:
        v = scores(logits, temperature, top_k, seed, pos, top_p)
        if nucleus_margin(logits, temperature, top_k, top_p) < NUCLEUS_EPS:
            ids = {int(np.argmax(scores(logits, temperature, top_k, seed, pos, top_p, d))) for d in (-1, 0, 1)}
            if len(ids) > 1:
                return 0.0
    top2 = np.partition(v, v.shape[0] - 2)[-2:]
    if not np.isfinite(top2).all():
        return float("inf")
    return float((top2[1] - top2[0]) / max(abs(float(top2[1])), 1.0))
