// The token-sampling rule: the one definition every kernel that turns logits into an id includes
// (kllm_sample_f32, the graph engine's argmax_advance_kernel, the persistent megakernel).  Its numpy
// mirror is kuiperllama_b200/sampling.py; DESIGN.md "Sampling" gives the reasons.
//
// Inputs: logits l[0..V) of position `pos`, temperature T, top_k k, 64-bit seed.
//   1. T == 0: greedy argmax (maximum, lowest index on ties) -- no noise is computed.
//   2. s_i = l_i / T, IEEE division.
//   3. 0 < k < V: tau = the k-th largest s_i; keep every i with s_i >= tau (ties at tau are kept).
//      k <= 0 or k >= V keeps everything.
//   4. Noise: Philox4x32-10, key (seed & 0xffffffff, seed >> 32).  Logit i takes word i & 3 of the
//      block at counter (i >> 2, pos, 0, 0); u = ((x >> 8) + 0.5) * 2^-24 rounded toward zero to fp32
//      (so u stays in (0, 1): the round-to-nearest of (2^24 - 0.5) * 2^-24 would be 1.0 and give an
//      infinite variate); g_i = -logf(-logf(u)).
//   5. id = argmax over kept i of (s_i + g_i), lowest index on ties.
// This is the Gumbel-max form of "softmax(s) over the kept set, then one multinomial draw".  The noise
// depends only on (seed, pos, i): the id is a pure function of the logits, the seed and the position,
// whichever engine or rank computes it.  Reusing a seed at the same position reuses the same noise.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace kllm {

// Device-resident sampling parameters (kllm_decoder_set_sampling).  Engines read them when they run,
// so changing them rebuilds nothing.  A zeroed struct is greedy.
struct SampleParams {
  float temperature;
  int32_t top_k;
  uint64_t seed;
};

namespace sampling {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
  constexpr uint32_t kM0 = 0xD2511F53u, kM1 = 0xCD9E8D57u, kW0 = 0x9E3779B9u, kW1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(kM0, c.x), lo0 = kM0 * c.x;
    const uint32_t hi1 = __umulhi(kM1, c.z), lo1 = kM1 * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += kW0;
    k.y += kW1;
  }
  return c;
}

__device__ __forceinline__ uint2 seed_key(uint64_t seed) {
  return make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
}

__device__ __forceinline__ uint32_t pick(const uint4& r, int w) {
  return w == 0 ? r.x : w == 1 ? r.y : w == 2 ? r.z : r.w;
}

__device__ __forceinline__ float gumbel(uint32_t x) {
  const float u = __fmul_rn(__fadd_rz(__uint2float_rn(x >> 8), 0.5f), 0x1p-24f);
  return -logf(-logf(u));
}

// s_i + g_i of logit i
__device__ __forceinline__ float perturbed(float l, float T, uint2 key, int pos, int i) {
  const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(i) >> 2, static_cast<uint32_t>(pos), 0u, 0u), key);
  return __fadd_rn(__fdiv_rn(l, T), gumbel(pick(r, i & 3)));
}

__device__ __forceinline__ bool top_k_active(const SampleParams& sp, int n) {
  return sp.temperature > 0.f && sp.top_k > 0 && sp.top_k < n;
}

// T > 0 without top-k: the id is a plain argmax of s_i + g_i, so the per-element values can be folded
// wherever the logits are produced, with the greedy reduction unchanged
__device__ __forceinline__ bool perturb_only(const SampleParams& sp, int n) {
  return sp.temperature > 0.f && !top_k_active(sp, n);
}

// (value, index): larger value wins, lowest index on ties -- the fold of the greedy argmax
__device__ __forceinline__ void fold(float& v, int& i, float ov, int oi) {
  if (oi >= 0 && (i < 0 || ov > v || (ov == v && oi < i))) {
    v = ov;
    i = oi;
  }
}

// Order-preserving map of fp32 onto uint32 (radix select)
__device__ __forceinline__ unsigned order_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k ^ 0x80000000u) : ~k);
}

// Shared-memory scratch of draw_block; the candidate list (cap pairs) follows it.
struct DrawScratch {
  unsigned hist[256];
  float red_v[32];
  int red_i[32];
  unsigned count, sel_digit, sel_above;
  int result;
  float lbound;
};
constexpr int kDrawScratchBase = static_cast<int>((sizeof(DrawScratch) + 15) & ~size_t{15});

// (v, i) of every thread of the block -> the winner, returned in every thread
template <int NT, class Sync>
__device__ __forceinline__ int block_fold(float v, int i, DrawScratch& s, Sync sync) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) fold(v, i, __shfl_down_sync(0xffffffffu, v, off), __shfl_down_sync(0xffffffffu, i, off));
  if (lane == 0) {
    s.red_v[warp] = v;
    s.red_i[warp] = i;
  }
  sync();
  if (warp == 0) {
    v = lane < NT / 32 ? s.red_v[lane] : 0.f;
    i = lane < NT / 32 ? s.red_i[lane] : -1;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) fold(v, i, __shfl_down_sync(0xffffffffu, v, off), __shfl_down_sync(0xffffffffu, i, off));
    if (lane == 0) s.result = i;
  }
  sync();
  return s.result;
}

// k-th largest of get(0..m) (1 <= k <= m): radix select over order_key, 8 bits per pass, from the top
template <int NT, class Get, class Sync>
__device__ __forceinline__ float kth_largest(Get get, int m, int k, DrawScratch& s, Sync sync) {
  const int tid = threadIdx.x, lane = tid & 31;
  unsigned prefix = 0u, mask = 0u, rem = static_cast<unsigned>(k);
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = tid; b < 256; b += NT) s.hist[b] = 0u;
    sync();
    for (int i0 = 0; i0 < m; i0 += NT) {
      const int i = i0 + tid;
      int bin = -1;
      if (i < m) {
        const unsigned key = order_key(get(i));
        if ((key & mask) == prefix) bin = static_cast<int>((key >> shift) & 255u);
      }
      // logits bunch into few bins: one shared atomic per distinct bin of the warp
      const unsigned peers = __match_any_sync(0xffffffffu, bin);
      if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(&s.hist[bin], static_cast<unsigned>(__popc(peers)));
    }
    sync();
    if (tid < 32) {  // lane l scans bins 255 - 8l down to 248 - 8l
      unsigned c[8], tot = 0u;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        c[j] = s.hist[255 - 8 * lane - j];
        tot += c[j];
      }
      unsigned inc = tot;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const unsigned o = __shfl_up_sync(0xffffffffu, inc, off);
        if (lane >= off) inc += o;
      }
      const int hit = __ffs(__ballot_sync(0xffffffffu, inc >= rem)) - 1;
      if (lane == hit) {
        unsigned above = inc - tot;
        bool found = false;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (!found && above + c[j] >= rem) {
            s.sel_digit = static_cast<unsigned>(255 - 8 * lane - j);
            s.sel_above = above;
            found = true;
          }
          if (!found) above += c[j];
        }
      }
    }
    sync();
    prefix |= s.sel_digit << shift;
    mask |= 0xffu << shift;
    rem -= s.sel_above;
  }
  return key_value(prefix);
}

// The rule, drawn by one block of NT threads over logits[0..n) (device memory, read through L2).  Returns
// the id in every thread.  `scratch` (16-byte aligned shared memory, scratch_bytes >= kDrawScratchBase)
// holds the histogram and a list of top-k candidates.
//
// Top-k without a full sort: a lower bound L of the k-th largest logit comes from the maxima of disjoint
// parts of the vector (k of them are k distinct logits >= L): `maxima` / `maxima_idx` (an index < 0
// marks an empty part) when the caller has them, else the block's per-thread maxima.  Only logits
// that can still reach tau after the division by T (l >= L less a few ulp) become candidates; tau and
// the kept argmax are then taken over the candidates in shared memory.  When they do not fit, the
// same selection runs over the whole vector instead.
template <int NT, class Sync>
__device__ __forceinline__ int draw_block(const float* logits, int n, const SampleParams sp, int pos,
                                          const float* maxima, const int* maxima_idx, int n_maxima,
                                          unsigned char* scratch, int scratch_bytes, Sync sync) {
  const int tid = threadIdx.x, lane = tid & 31;
  DrawScratch& s = *reinterpret_cast<DrawScratch*>(scratch);
  const int cap = (scratch_bytes - kDrawScratchBase) / 8;
  float* cand_s = reinterpret_cast<float*>(scratch + kDrawScratchBase);
  int* cand_i = reinterpret_cast<int*>(cand_s + cap);
  const float T = sp.temperature;
  float bv = 0.f;
  int bi = -1;
  if (!(T > 0.f)) {  // greedy (argmax_kernel.cu:49-71 semantics)
    for (int i = tid; i < n; i += NT) {
      const float v = __ldcg(logits + i);
      if (bi < 0 || v > bv) {
        bv = v;
        bi = i;
      }
    }
    return block_fold<NT>(bv, bi, s, sync);
  }
  const uint2 key = seed_key(sp.seed);
  if (!top_k_active(sp, n)) {  // one Philox block serves four consecutive logits
    for (int j = tid; j < ((n + 3) >> 2); j += NT) {
      const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(j), static_cast<uint32_t>(pos), 0u, 0u), key);
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const int i = 4 * j + w;
        if (i < n) fold(bv, bi, __fadd_rn(__fdiv_rn(__ldcg(logits + i), T), gumbel(pick(r, w))), i);
      }
    }
    return block_fold<NT>(bv, bi, s, sync);
  }

  // ---- top-k: lower bound L of the k-th largest logit ----
  const int k = sp.top_k;
  if (maxima == nullptr) {  // per-thread maxima (cap >= NT)
    float mx = -INFINITY;
    for (int i = tid; i < n; i += NT) mx = fmaxf(mx, __ldcg(logits + i));
    cand_s[tid] = mx;
    n_maxima = NT;
  }
  if (tid == 0) {
    s.lbound = -INFINITY;
    s.count = 0u;
  }
  sync();
  auto max_at = [&](int j) {
    if (maxima == nullptr) return cand_s[j];
    return maxima_idx[j] < 0 ? -INFINITY : __ldcg(maxima + j);
  };
  if (k <= n_maxima) {  // L = the maximum with exactly k - 1 ahead of it (larger, or equal and earlier)
    for (int t = tid; t < n_maxima; t += NT) {
      const float v = max_at(t);
      int ahead = 0;
      for (int j = 0; j < n_maxima; ++j) {
        const float w = max_at(j);
        ahead += (w > v || (w == v && j < t)) ? 1 : 0;
      }
      if (ahead == k - 1) s.lbound = v;
    }
  }
  sync();
  const float L = s.lbound;
  // l < L can still give l / T == L / T after rounding: admit everything within 2^-20 relative of L
  const float lo = isfinite(L) ? L - (fabsf(L) * 0x1p-20f + T * 0x1p-126f) : -INFINITY;

  // ---- candidates: kUnroll independent L2 loads in flight per thread, then the warp-aggregated appends ----
  constexpr int kUnroll = 16;
  for (int i0 = 0; i0 < n; i0 += NT * kUnroll) {
    float l[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int i = i0 + u * NT + tid;
      l[u] = i < n ? __ldcg(logits + i) : -INFINITY;
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const int i = i0 + u * NT + tid;
      const bool c = i < n && l[u] >= lo;
      const unsigned ball = __ballot_sync(0xffffffffu, c);
      if (ball == 0u) continue;
      unsigned base = 0u;
      if (lane == 0) base = atomicAdd(&s.count, static_cast<unsigned>(__popc(ball)));
      base = __shfl_sync(0xffffffffu, base, 0);
      const int slot = static_cast<int>(base) + __popc(ball & ((1u << lane) - 1u));
      if (c && slot < cap) {
        cand_s[slot] = __fdiv_rn(l[u], T);
        cand_i[slot] = i;
      }
    }
  }
  sync();
  const int m = static_cast<int>(s.count);
  if (m <= cap) {
    const float tau = kth_largest<NT>([&](int c) { return cand_s[c]; }, m, k, s, sync);
    for (int c = tid; c < m; c += NT) {
      const float sv = cand_s[c];
      if (sv >= tau) {
        const int i = cand_i[c];
        const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(i) >> 2, static_cast<uint32_t>(pos), 0u, 0u), key);
        fold(bv, bi, __fadd_rn(sv, gumbel(pick(r, i & 3))), i);
      }
    }
  } else {  // too many candidates for the scratch: the same selection over the whole vector
    const float tau = kth_largest<NT>([&](int i) { return __fdiv_rn(__ldcg(logits + i), T); }, n, k, s, sync);
    for (int i = tid; i < n; i += NT) {
      const float l = __ldcg(logits + i);
      if (__fdiv_rn(l, T) >= tau) fold(bv, bi, perturbed(l, T, key, pos, i), i);
    }
  }
  return block_fold<NT>(bv, bi, s, sync);
}

}  // namespace sampling
}  // namespace kllm
