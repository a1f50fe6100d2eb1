// The token-sampling rule: the one definition every kernel that turns logits into an id includes
// (kllm_sample_f32, the graph engine's argmax_advance_kernel, the persistent megakernel).  Its numpy
// mirror is kuiperllama_b200/sampling.py; DESIGN.md "Sampling" gives the reasons.
//
// Inputs: logits l[0..V) of position `pos`, temperature T, top_k k, top_p, 64-bit seed, repetition penalty
// theta with window last_n, and the history H(pos) of fed ids.
//   0. History: H(pos) = the ids fed as input at positions j in [lo, pos], lo = 0 for last_n == 0 (the whole
//      sequence) else max(0, pos - last_n + 1).  "Fed at j" is the id whose embedding entered the model at
//      position j (its K/V rows are row j of the cache), by whichever entry fed it; a position never fed, or
//      fed an id outside [0, V), holds none.  Feeding a position again overwrites it.
//  0b. Repetition penalty (HF's RepetitionPenaltyLogitsProcessor): for i in H(pos),
//      l'_i = l_i < 0 ? l_i * theta : l_i / theta (one fp32 IEEE multiply or divide); every other l'_i = l_i.
//      An id that occurs more than once is penalised once.  theta == 1 is off.
//   Step 0 runs as four sub-steps, in HF's order (sequence bias before the repetition penalty) and, within the
//   penalties, vLLM's (repetition, frequency, presence), each one fp32 IEEE operation:
//  0a. Logit bias: l_i + b_i for every i, b the dense [V] table of an {id: bias} map (unset entries 0, each
//      entry 0 + bias as HF builds it).  Skipped when no bias is set, which keeps the sign of a -0.0 logit.
//  0b. The repetition penalty above, over H(pos).
//  0c. Frequency: C(pos) = the multiset of ids fed at positions [from_pos, pos] (empty for from_pos > pos), c_i
//      the multiplicity of i in it.  For c_i > 0: l_i - alpha_f * (float)c_i.  Skipped for alpha_f == 0.
//  0d. Presence: for c_i > 0, l_i - alpha_p.  Skipped for alpha_p == 0.
//   With every sub-step off the history is not read.  Counts are exact integers, so every block, CTA, engine
//   and rank computes the same l'.  Steps 1 to 5 run on l'.
//   1. T == 0: greedy argmax (maximum, lowest index on ties) -- no noise is computed.
//   2. s_i = l_i / T, IEEE division.
//   3. 0 < k < V: tau = the k-th largest s_i; keep every i with s_i >= tau (ties at tau are kept).
//      k <= 0 or k >= V keeps everything.
//  3b. 0 < top_p < 1 (nucleus): K = the set kept by step 3, m = max over K of s_i.  Mass
//      q_i = floor(expf(s_i - m) * 2^32) (fp32 weight, so the maximum's mass is 2^32 and a weight below 2^-32
//      is mass 0); Z = sum over K of q_i and A_i = sum over K of q_j with s_j > s_i, both exact uint64.
//      p24 = max(1, rint(top_p * 2^24)).  Keep i iff A_i * 2^24 < p24 * Z (exact, 128-bit): HF's "drop a
//      token once the mass strictly above it reaches p", with equal s kept or dropped together.  The kept
//      set is {s_i >= tau_p}; it always holds the maximum.  Integer sums do not depend on their order, so
//      every block, engine and rank finds the same tau_p.
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
#include <type_traits>

namespace kllm {

// Sampling parameters (kllm_decoder_set_sampling_top_p).  A zeroed struct is greedy (and top_p 0 is off, as is 1).
struct SampleParams {
  float temperature;
  int32_t top_k;
  uint64_t seed;
  float top_p;
};

// Step 0 (kllm_decoder_set_repetition_penalty, kllm_decoder_set_frequency_presence, kllm_decoder_set_logit_bias).
// A zeroed struct is off.  `active` is set by the host (step0_finish) when any sub-step is on, so that the
// engines test one word.  `marks` [V] is zero between tokens (step0_rows).
struct PenaltyParams {
  int32_t active;
  float penalty;      // 0b; 1 (or 0 in a zeroed struct) is off
  int32_t last_n;     // 0b's window
  float frequency;    // 0c; 0 is off
  float presence;     // 0d; 0 is off
  int32_t from_pos;   // 0c / 0d count the ids fed at [from_pos, pos]
  const float* bias;  // 0a's dense [V] table; null is off
  int32_t* marks;
};

// Everything a decoder's ids are drawn and recorded under: its setters change a copy and put it in force between
// two stream synchronises, on the host and in one device copy that the engines read (decoder.cu put_settings).
struct DrawSettings {
  SampleParams sample;
  PenaltyParams penalty;
  int32_t lp_top_n;  // log-probabilities: -1 off; 0 the id's lp; 1..kMaxTopLogprobs also the top-N (DESIGN.md 5.8)
};

namespace sampling {

__host__ __device__ __forceinline__ bool penalty_active(const PenaltyParams& pp) {
  return pp.penalty > 0.f && pp.penalty != 1.f;
}

__host__ __device__ __forceinline__ bool counts_active(const PenaltyParams& pp) {
  return pp.frequency != 0.f || pp.presence != 0.f;
}

// The host's last word on a PenaltyParams it changed
__host__ __forceinline__ void step0_finish(PenaltyParams& pp) {
  pp.active = penalty_active(pp) || counts_active(pp) || pp.bias != nullptr;
}

__host__ __device__ __forceinline__ bool step0_active(const PenaltyParams& pp) { return pp.active != 0; }

// Step 0's lower end of the window at `pos`
__host__ __device__ __forceinline__ int window_lo(const PenaltyParams& pp, int pos) {
  return pp.last_n == 0 ? 0 : max(0, pos - pp.last_n + 1);
}

// Step 0b on one logit of the history
__device__ __forceinline__ float penalize(float l, float theta) {
  return l < 0.f ? __fmul_rn(l, theta) : __fdiv_rn(l, theta);
}

// A mark word of step0_rows: bit 30 is membership in H(pos), bits 0..29 the count c_i (positions < 2^30)
constexpr int32_t kInHistory = 1 << 30;

// The whole of step 0 on the raw logit l of id i with mark word `mark`
__device__ __forceinline__ float step0_value(float l, const PenaltyParams& pp, int i, int32_t mark) {
  if (pp.bias != nullptr) l = __fadd_rn(l, __ldg(pp.bias + i));
  if (mark & kInHistory) l = penalize(l, pp.penalty);
  if (mark & (kInHistory - 1)) {
    if (pp.frequency != 0.f) l = __fsub_rn(l, __fmul_rn(pp.frequency, __int2float_rn(mark & (kInHistory - 1))));
    if (pp.presence != 0.f) l = __fsub_rn(l, pp.presence);
  }
  return l;
}

// ids[lo, hi): step 0's windows are two such ranges of the history
struct IdRange {
  const int32_t* ids;
  int lo, hi;
};

// fn(id) for the entries j of r with j = t (mod NT), t this thread
template <int NT, class F>
__device__ __forceinline__ void for_each_id(const IdRange& r, F fn) {
  const int tid = threadIdx.x;
  for (int j = r.lo + ((tid - r.lo % NT) + NT) % NT; j < r.hi; j += NT) fn(__ldcg(r.ids + j));
}

// Step 0 of logits[lo_row, hi_row) into out[lo_row, hi_row) by the NT threads of one block (or one CTA's
// consumer threads), `rep` the ids of H(pos) and `cnt` those of C(pos):
//   1. the copy pass writes l_i (+ b_i);
//   2. every id of either window in the row range is marked in pp.marks with integer atomics: + 1 per
//      occurrence in `cnt`, | kInHistory for one in `rep`;
//   3. every thread that meets an id writes step0_value of its raw logit and its mark word, so a duplicate
//      writes the same value again and no deduplication is needed;
//   4. the marks of the ids met are reset to 0.
// Thread t reads the window entries j = t (mod NT) only.  Rows outside [lo_row, hi_row) are not touched, so
// blocks over disjoint ranges do not race.  `sync` orders each pass before the next (a CTA barrier orders
// global memory between its threads) and the writes before the caller's reads; the reset needs no barrier of
// its own, as the next token's marks come behind the caller's.
template <int NT, class Sync>
__device__ __forceinline__ void step0_rows(const float* logits, float* out, int lo_row, int hi_row,
                                           const PenaltyParams& pp, const IdRange& rep, const IdRange& cnt,
                                           Sync sync) {
  const int tid = threadIdx.x;
  for (int i = lo_row + tid; i < hi_row; i += NT) {
    const float l = __ldcg(logits + i);
    out[i] = pp.bias != nullptr ? __fadd_rn(l, __ldg(pp.bias + i)) : l;
  }
  if (rep.lo >= rep.hi && cnt.lo >= cnt.hi) {  // the bias alone
    sync();
    return;
  }
  int32_t* marks = pp.marks;
  const auto mine = [lo_row, hi_row](int id) { return id >= lo_row && id < hi_row; };
  for_each_id<NT>(cnt, [&](int id) { if (mine(id)) atomicAdd(marks + id, 1); });
  for_each_id<NT>(rep, [&](int id) { if (mine(id)) atomicOr(marks + id, kInHistory); });
  sync();
  const auto write = [&](int id) {
    if (mine(id)) out[id] = step0_value(__ldcg(logits + id), pp, id, __ldcg(marks + id));
  };
  for_each_id<NT>(cnt, write);
  for_each_id<NT>(rep, write);
  sync();
  const auto reset = [&](int id) { if (mine(id)) marks[id] = 0; };
  for_each_id<NT>(cnt, reset);
  for_each_id<NT>(rep, reset);
}

// Step 0 at `pos` over the decoder's history hist[seq_len] (the id fed at each position)
template <int NT, class Sync>
__device__ __forceinline__ void step0_history(const float* logits, float* out, int lo_row, int hi_row,
                                              const PenaltyParams& pp, const int32_t* hist, int pos, Sync sync) {
  const IdRange rep{hist, penalty_active(pp) ? window_lo(pp, pos) : 0, penalty_active(pp) ? pos + 1 : 0};
  const IdRange cnt{hist, counts_active(pp) ? max(0, pp.from_pos) : 0, counts_active(pp) ? pos + 1 : 0};
  step0_rows<NT>(logits, out, lo_row, hi_row, pp, rep, cnt, sync);
}

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

__device__ __forceinline__ bool top_p_active(const SampleParams& sp) {
  return sp.temperature > 0.f && sp.top_p > 0.f && sp.top_p < 1.f;
}

// T > 0 without top-k or top-p: the id is a plain argmax of s_i + g_i, so the per-element values can be
// folded wherever the logits are produced, with the greedy reduction unchanged
__device__ __forceinline__ bool perturb_only(const SampleParams& sp, int n) {
  return sp.temperature > 0.f && !top_k_active(sp, n) && !top_p_active(sp);
}

// Top-k or top-p: the kept set needs a threshold over the whole vector, so one block draws the id
__device__ __forceinline__ bool needs_draw(const SampleParams& sp, int n) {
  return top_k_active(sp, n) || top_p_active(sp);
}

// Step 3b's mass of score s under the kept maximum m: floor(expf(s - m) * 2^32), at most 2^32
__device__ __forceinline__ unsigned long long nucleus_mass(float s, float m) {
  return __float2ull_rz(__fmul_rn(expf(__fsub_rn(s, m)), 0x1p32f));
}

// ceil(p24 * Z / 2^24): a token is kept iff the mass strictly above it is below this, so tau_p is the
// largest s whose mass at or above it reaches it (p24 * Z < 2^74: the 128-bit product, then the shift)
__device__ __forceinline__ unsigned long long nucleus_need(unsigned long long Z, float top_p) {
  const unsigned long long p24 = max(1ull, static_cast<unsigned long long>(rintf(__fmul_rn(top_p, 0x1p24f))));
  const unsigned long long lo = p24 * Z, hi = __umul64hi(p24, Z);
  return ((hi << 40) | (lo >> 24)) + ((lo & 0xffffffull) != 0ull ? 1ull : 0ull);
}

// The bin of a score in the nucleus's first pass: 8 bins per unit of m - s, from the top; every token
// with nonzero mass (m - s <= 22.2) lies in the first 178
__device__ __forceinline__ int nucleus_bin(float s, float m) {
  return 255 - min(255, static_cast<int>(__fmul_rn(__fsub_rn(m, s), 8.f)));
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
  union {
    unsigned hist[256];              // counts (top-k)
    unsigned long long mass[256];    // masses (top-p)
  };
  unsigned long long sel_above, total;
  unsigned long long red_q[32];
  float red_v[32];
  int red_i[32];
  unsigned count, sel_digit;
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

// Histogram scan of the selects: bins from 255 down, the first at which the running weight reaches
// need(total) -> s.sel_digit, the weight of the bins before it -> s.sel_above, the total -> s.total.
// Run by warp 0.
template <class W, class Need>
__device__ __forceinline__ void scan_bins(const W* hist, Need need, DrawScratch& s) {
  const int lane = threadIdx.x & 31;
  W c[8], tot = 0;  // lane l scans bins 255 - 8l down to 248 - 8l
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    c[j] = hist[255 - 8 * lane - j];
    tot += c[j];
  }
  W inc = tot;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const W o = __shfl_up_sync(0xffffffffu, inc, off);
    if (lane >= off) inc += o;
  }
  const W total = __shfl_sync(0xffffffffu, inc, 31);
  const W rem = need(total);
  const int hit = __ffs(__ballot_sync(0xffffffffu, inc >= rem)) - 1;
  if (lane == hit) {
    W above = inc - tot;
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
  if (lane == 0) s.total = total;
}

// The largest value v of get(0..m) whose weight at or above v reaches `need` (0 < need <= total weight):
// radix select over order_key, 8 bits per pass, from the top.  W = unsigned counts (weight 1 each) gives
// the k-th largest; W = unsigned long long gives step 3b's tau_p with the nucleus masses as weights.
template <int NT, class W, class Get, class Weight, class Sync>
__device__ __forceinline__ float select_top(Get get, Weight weight, int m, W need, DrawScratch& s, Sync sync) {
  constexpr bool kCount = std::is_same<W, unsigned>::value;
  W* hist = reinterpret_cast<W*>(kCount ? static_cast<void*>(s.hist) : static_cast<void*>(s.mass));
  const int tid = threadIdx.x, lane = tid & 31;
  unsigned prefix = 0u, mask = 0u;
  W rem = need;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = tid; b < 256; b += NT) hist[b] = 0;
    sync();
    for (int i0 = 0; i0 < m; i0 += NT) {
      const int i = i0 + tid;
      int bin = -1;
      if (i < m) {
        const unsigned key = order_key(get(i));
        if ((key & mask) == prefix) bin = static_cast<int>((key >> shift) & 255u);
      }
      if constexpr (kCount) {
        // logits bunch into few bins: one shared atomic per distinct bin of the warp
        const unsigned peers = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], static_cast<unsigned>(__popc(peers)));
      } else {
        W w = bin >= 0 ? weight(i) : W(0);
        // flat distributions put whole warps into one bin: one atomic for the warp's sum then
        if (__match_any_sync(0xffffffffu, bin) == 0xffffffffu) {
#pragma unroll
          for (int off = 16; off > 0; off >>= 1) w += __shfl_xor_sync(0xffffffffu, w, off);
          if (lane == 0 && bin >= 0 && w != 0) atomicAdd(&hist[bin], w);
        } else if (w != 0) {
          atomicAdd(&hist[bin], w);
        }
      }
    }
    sync();
    if (tid < 32) scan_bins<W>(hist, [rem](W) { return rem; }, s);
    sync();
    prefix |= s.sel_digit << shift;
    mask |= 0xffu << shift;
    rem -= static_cast<W>(s.sel_above);
  }
  return key_value(prefix);
}

// k-th largest of get(0..m) (1 <= k <= m)
template <int NT, class Get, class Sync>
__device__ __forceinline__ float kth_largest(Get get, int m, int k, DrawScratch& s, Sync sync) {
  return select_top<NT, unsigned>(get, [](int) { return 1u; }, m, static_cast<unsigned>(k), s, sync);
}

// Sum of v over the block, returned in every thread
template <int NT, class Sync>
__device__ __forceinline__ unsigned long long block_sum(unsigned long long v, DrawScratch& s, Sync sync) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
  if (lane == 0) s.red_q[warp] = v;
  sync();
  unsigned long long t = 0ull;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) t += s.red_q[w];
  sync();
  return t;
}

// The rule, drawn by one block of NT threads over logits[0..n) (device memory, read through L2).  Returns
// the id in every thread.  `scratch` (16-byte aligned shared memory, scratch_bytes >= kDrawScratchBase)
// holds the histogram and a list of candidates.
//
// Top-k without a full sort: a lower bound L of the k-th largest logit comes from the maxima of disjoint
// parts of the vector (k of them are k distinct logits >= L): `maxima` / `maxima_idx` (an index < 0
// marks an empty part) when the caller has them, else the block's per-thread maxima.  Only logits
// that can still reach tau after the division by T (l >= L less a few ulp) become candidates; tau and
// the kept argmax are then taken over the candidates in shared memory.
//
// Top-p with top-k runs step 3b over the top-k candidates.  Top-p alone takes the maximum from the same
// maxima (else one more pass).  One pass then sums the masses into 256 bins of 1/8 of m - s (Z, and the
// first bins whose mass reaches the need, which bound tau_p from below) and collects the scores within 8 of
// m.  When the nucleus reaches below those, or they do not fit, a second pass collects the logits of the
// bins from the one where the mass reaches the need.  tau_p is the mass-weighted select over the candidates.
//
// When the candidates do not fit, the same selections run over the whole vector instead.
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
  const bool tk = top_k_active(sp, n), tp = top_p_active(sp);
  if (!tk && !tp) {  // one Philox block serves four consecutive logits
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

  // f(l, i, valid) over the whole vector, kUnroll independent L2 loads in flight per thread; every lane
  // calls f the same number of times (f may use warp votes)
  constexpr int kUnroll = 16;
  auto for_each_logit = [&](auto f) {
    for (int i0 = 0; i0 < n; i0 += NT * kUnroll) {
      float l[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const int i = i0 + u * NT + tid;
        l[u] = i < n ? __ldcg(logits + i) : -INFINITY;
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) f(l[u], i0 + u * NT + tid, i0 + u * NT + tid < n);
    }
  };
  // the block's maximum logit, by a pass over the vector
  auto max_logit = [&]() {
    float v = 0.f;
    int vi = -1;
    for (int i = tid; i < n; i += NT) fold(v, vi, __ldcg(logits + i), i);
    return __ldcg(logits + block_fold<NT>(v, vi, s, sync));
  };

  float mx = 0.f;                    // m of step 3b (top-p alone: known before the candidates are taken)
  unsigned long long need = 0ull;    // nucleus_need(Z) (likewise)
  float lo = -INFINITY;              // the candidates are logits l >= lo (and more conditions for top-p alone)
  if (tid == 0) s.count = 0u;        // (published by the barriers of either branch)
  if (tk) {
    // ---- top-k: lower bound L of the k-th largest logit ----
    const int k = sp.top_k;
    if (maxima == nullptr) {  // per-thread maxima (cap >= NT)
      float mxl = -INFINITY;
      for (int i = tid; i < n; i += NT) mxl = fmaxf(mxl, __ldcg(logits + i));
      cand_s[tid] = mxl;
      n_maxima = NT;
    }
    if (tid == 0) s.lbound = -INFINITY;
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
    lo = isfinite(L) ? L - (fabsf(L) * 0x1p-20f + T * 0x1p-126f) : -INFINITY;
  } else {
    // ---- top-p alone: the maximum (from the parts' maxima when the caller has them) ----
    float lmax;
    if (maxima != nullptr) {
      for (int j = tid; j < n_maxima; j += NT)
        if (maxima_idx[j] >= 0) fold(bv, bi, __ldcg(maxima + j), j);
      lmax = __ldcg(maxima + block_fold<NT>(bv, bi, s, sync));
      bv = 0.f;
      bi = -1;
    } else {
      lmax = max_logit();
    }
    mx = __fdiv_rn(lmax, T);
    // raw logits below this have s < m - 23, mass 0 (expf(-23) 2^32 < 1): skipped without the division
    lo = lmax - (23.f * T + (fabsf(lmax) + 23.f * T) * 0x1p-16f);
  }

  // ---- candidates (s, i) = (l / T, i): warp-aggregated appends (beyond cap: counted, not stored) ----
  auto append = [&](bool c, float sv, int i) {
    const unsigned ball = __ballot_sync(0xffffffffu, c);
    if (ball == 0u) return;
    unsigned base = 0u;
    if (lane == 0) base = atomicAdd(&s.count, static_cast<unsigned>(__popc(ball)));
    base = __shfl_sync(0xffffffffu, base, 0);
    const int slot = static_cast<int>(base) + __popc(ball & ((1u << lane) - 1u));
    if (c && slot < cap) {
      cand_s[slot] = sv;
      cand_i[slot] = i;
    }
  };
  // one pass: the logits l >= lo with keep(l) become candidates; returns their count
  auto collect = [&](auto keep) {
    for_each_logit([&](float l, int i, bool valid) {
      const bool c = valid && l >= lo && keep(l);
      append(c, c ? __fdiv_rn(l, T) : 0.f, i);
    });
    sync();
    return static_cast<int>(s.count);
  };
  int m;
  if (tk) {
    m = collect([](float) { return true; });
  } else {
    // ---- top-p alone, one pass: the masses into 256 bins of 1/8 of m - s (Z, and the first bins whose
    // mass reaches the need), while the scores within 8 of m become candidates ----
    constexpr int kNearBin = 255 - 64;
    for (int b = tid; b < 256; b += NT) s.mass[b] = 0ull;
    sync();
    for_each_logit([&](float l, int i, bool valid) {
      float sv = 0.f;
      int bin = -1;
      unsigned long long q = 0ull;
      if (valid && l >= lo) {
        sv = __fdiv_rn(l, T);
        if (__fsub_rn(mx, sv) < 23.f) {
          q = nucleus_mass(sv, mx);
          bin = nucleus_bin(sv, mx);
        }
      }
      if (__match_any_sync(0xffffffffu, bin) == 0xffffffffu) {  // a flat stretch: one atomic per warp
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
        if (lane == 0 && q != 0ull) atomicAdd(&s.mass[bin], q);
      } else if (q != 0ull) {
        atomicAdd(&s.mass[bin], q);
      }
      append(bin >= kNearBin, sv, i);
    });
    sync();
    if (tid < 32) scan_bins<unsigned long long>(s.mass, [&](unsigned long long Z) { return nucleus_need(Z, sp.top_p); }, s);
    sync();
    const int top_bin = static_cast<int>(s.sel_digit);
    need = nucleus_need(s.total, sp.top_p);
    m = static_cast<int>(s.count);
    if (top_bin < kNearBin || m > cap) {
      // the nucleus reaches below the candidates, or they overflowed: a second pass collects the bins
      // from the one where the mass reaches the need
      sync();
      if (tid == 0) s.count = 0u;
      sync();
      m = collect([&](float l) { return nucleus_bin(__fdiv_rn(l, T), mx) >= top_bin; });
    }
  }
  if (m <= cap) {
    auto cand = [&](int c) { return cand_s[c]; };
    const float tau_k = tk ? kth_largest<NT>(cand, m, sp.top_k, s, sync) : -INFINITY;
    float tau = tau_k;
    if (tp) {
      if (tk) {  // step 3b over the top-k candidates: their maximum and Z
        for (int c = tid; c < m; c += NT) fold(bv, bi, cand_s[c], c);
        mx = cand_s[block_fold<NT>(bv, bi, s, sync)];
        bv = 0.f;
        bi = -1;
        unsigned long long z = 0ull;
        for (int c = tid; c < m; c += NT)
          if (cand_s[c] >= tau_k) z += nucleus_mass(cand_s[c], mx);
        need = nucleus_need(block_sum<NT>(z, s, sync), sp.top_p);
      }
      tau = select_top<NT, unsigned long long>(
          cand, [&](int c) { return cand_s[c] >= tau_k ? nucleus_mass(cand_s[c], mx) : 0ull; }, m, need, s, sync);
    }
    for (int c = tid; c < m; c += NT) {
      const float sv = cand_s[c];
      if (sv >= tau) {
        const int i = cand_i[c];
        const uint4 r = philox4x32_10(make_uint4(static_cast<uint32_t>(i) >> 2, static_cast<uint32_t>(pos), 0u, 0u), key);
        fold(bv, bi, __fadd_rn(sv, gumbel(pick(r, i & 3))), i);
      }
    }
  } else {  // too many candidates for the scratch: the same selections over the whole vector
    auto score = [&](int i) { return __fdiv_rn(__ldcg(logits + i), T); };
    const float tau_k = tk ? kth_largest<NT>(score, n, sp.top_k, s, sync) : -INFINITY;
    float tau = tau_k;
    if (tp) {
      if (tk) {
        mx = __fdiv_rn(max_logit(), T);
        unsigned long long z = 0ull;
        for (int i = tid; i < n; i += NT) {
          const float sv = score(i);
          if (sv >= tau_k) z += nucleus_mass(sv, mx);
        }
        need = nucleus_need(block_sum<NT>(z, s, sync), sp.top_p);
      }
      tau = select_top<NT, unsigned long long>(
          score, [&](int i) { const float sv = score(i); return sv >= tau_k ? nucleus_mass(sv, mx) : 0ull; }, n, need,
          s, sync);
    }
    for (int i = tid; i < n; i += NT) {
      const float l = __ldcg(logits + i);
      if (__fdiv_rn(l, T) >= tau) fold(bv, bi, perturbed(l, T, key, pos, i), i);
    }
  }
  return block_fold<NT>(bv, bi, s, sync);
}

// ---- log-probabilities (DESIGN.md 5.8) ------------------------------------------------------------------
// Over the RAW logits l[0..V) of position pos (what kllm_decoder_logits returns: before step 0b, temperature,
// top-k and top-p), for a partition of [0, V) into parts:
//  L1. For each part c: m_c = max of its l_i; S_c = sum of expf(l_i - m_c) over its l_i, in fp32.
//  L2. m = max over the parts of m_c; S = sum over c of S_c * expf(m_c - m), folded in part-index order;
//      lse_off = logf(S).
//  L3. lp_i = (l_i - m) - lse_off, two IEEE fp32 subtractions.
//  Top-N: the N largest l_i in descending order, lowest index on ties (the greedy fold's order), each with its
//  lp_i.  A selection has no rounding, so the ids are exact whatever the partition.
// The same partition gives the same bits (every run, CTA and tensor-parallel rank); different partitions agree
// within the bound of DESIGN.md 5.8.  Parts: a CTA's classifier rows (or its range of the tensor-parallel gather)
// in the persistent engine, a warp's contiguous range in the one-block kernels.  Mirror: sampling.logprobs.
constexpr int kMaxTopLogprobs = 20;  // == KLLM_MAX_TOP_LOGPROBS

// The decoder's record, indexed by position: id[pos], lp[pos], top_ids / top_lp [pos][kMaxTopLogprobs]
struct LogprobRecord {
  int32_t* id;
  float* lp;
  int32_t* top_ids;
  float* top_lp;
};

struct Cand {
  float v;
  int i;  // < 0: no entry
};

// L3
__device__ __forceinline__ float logprob(float l, float m, float lse_off) { return __fsub_rn(__fsub_rn(l, m), lse_off); }

// Sum over a warp by a fixed butterfly: every lane ends with the same bits
__device__ __forceinline__ float warp_sum_fixed(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}

// Shared memory of the logprob routines, in front of top_n_block's scratch
struct LogprobScratch {
  float part_m[32], part_s[32];  // per-warp partials
  float m, lse_off;
  float top_v[kMaxTopLogprobs];
  int top_i[kMaxTopLogprobs];
};
constexpr int kLogprobScratchBase = static_cast<int>((sizeof(LogprobScratch) + 15) & ~size_t{15});
// scratch bytes the logprob routines of a block of NT threads need (top_n_block keeps NT maxima)
__host__ __device__ constexpr int logprob_scratch_bytes(int NT) { return kLogprobScratchBase + kDrawScratchBase + NT * 8; }

// L1 of the part get(lo..hi) by one warp, in every lane: lane j takes i = lo + j (mod 32) in increasing order,
// then the fixed butterfly
template <class Get>
__device__ __forceinline__ float2 warp_part(Get get, int lo, int hi) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int i = lo + lane; i < hi; i += 32) mx = fmaxf(mx, get(i));
  mx = warp_max(mx);
  float s = 0.f;
  for (int i = lo + lane; i < hi; i += 32) s = __fadd_rn(s, expf(__fsub_rn(get(i), mx)));
  return make_float2(mx, warp_sum_fixed(s));
}

// L1 of the part get(lo..hi) by a block of NT threads, returned in thread 0: thread t takes i = lo + t (mod NT) in
// increasing order, the fixed butterfly per warp, then the warp sums in warp order
template <int NT, class Get, class Sync>
__device__ __forceinline__ float2 block_part(Get get, int lo, int hi, LogprobScratch& ls, Sync sync) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float mx = -INFINITY;
  for (int i = lo + tid; i < hi; i += NT) mx = fmaxf(mx, get(i));
  mx = warp_max(mx);
  if (lane == 0) ls.part_m[warp] = mx;
  sync();
  mx = -INFINITY;
#pragma unroll
  for (int w = 0; w < NT / 32; ++w) mx = fmaxf(mx, ls.part_m[w]);
  float s = 0.f;
  if (mx > -INFINITY)
    for (int i = lo + tid; i < hi; i += NT) s = __fadd_rn(s, expf(__fsub_rn(get(i), mx)));
  s = warp_sum_fixed(s);
  if (lane == 0) ls.part_s[warp] = s;
  sync();
  s = 0.f;
  if (tid == 0)
    for (int w = 0; w < NT / 32; ++w) s = __fadd_rn(s, ls.part_s[w]);
  return make_float2(mx, s);
}

// L2 over parts part(0..n_parts) -> (m, lse_off) in every lane of the calling warp.  Lane 0 folds in part order.
template <class Part>
__device__ __forceinline__ float2 warp_fold_parts(Part part, int n_parts) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int c = lane; c < n_parts; c += 32) mx = fmaxf(mx, part(c).x);
  mx = warp_max(mx);
  float s = 0.f;
  if (lane == 0)
    for (int c = 0; c < n_parts; ++c) {
      const float2 p = part(c);
      if (p.y > 0.f) s = __fadd_rn(s, __fmul_rn(p.y, expf(__fsub_rn(p.x, mx))));
    }
  return make_float2(mx, logf(__shfl_sync(0xffffffffu, s, 0)));
}

// Top-N of get(0..m) (get(k) -> Cand; entries with i < 0 are skipped) by one warp, written to out_v / out_i[0..N)
// by lane 0; index -1 (lp -inf) pads a list with fewer than N entries.  Round r takes the best entry that ranks
// after round r - 1's.
template <class Get>
__device__ __forceinline__ void warp_top_n(Get get, int m, int N, float* out_v, int* out_i) {
  const int lane = threadIdx.x & 31;
  float pv = 0.f;
  int pi = -1;
  bool more = true;
  for (int r = 0; r < N; ++r) {
    float bv = 0.f;
    int bi = -1;
    if (more)
      for (int k = lane; k < m; k += 32) {
        const Cand c = get(k);
        if (c.i >= 0 && (r == 0 || c.v < pv || (c.v == pv && c.i > pi))) fold(bv, bi, c.v, c.i);
      }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) fold(bv, bi, __shfl_xor_sync(0xffffffffu, bv, off), __shfl_xor_sync(0xffffffffu, bi, off));
    if (lane == 0) {
      out_v[r] = bi < 0 ? -INFINITY : bv;
      out_i[r] = bi;
    }
    more = bi >= 0;
    pv = bv;
    pi = bi;
  }
}

// Top-N of get(0..m) by a block of NT threads into out_v / out_i[0..N) (visible to the block on return).
// scratch: logprob_scratch_bytes(NT) - kLogprobScratchBase bytes or more.  A lower bound tau of the N-th largest
// value is the N-th largest of the NT per-thread maxima (N distinct entries reach it), so only the entries >= tau
// become candidates; when they do not fit the scratch, the warp's rounds run over the whole list instead.
template <int NT, class Get, class Sync>
__device__ __forceinline__ void top_n_block(Get get, int m, int N, unsigned char* scratch, int scratch_bytes,
                                            float* out_v, int* out_i, Sync sync) {
  const int tid = threadIdx.x, lane = tid & 31;
  DrawScratch& s = *reinterpret_cast<DrawScratch*>(scratch);
  const int cap = (scratch_bytes - kDrawScratchBase) / 8;
  float* cv = reinterpret_cast<float*>(scratch + kDrawScratchBase);
  int* ci = reinterpret_cast<int*>(cv + cap);
  float bv = 0.f;
  int bi = -1;
  for (int k = tid; k < m; k += NT) {
    const Cand c = get(k);
    fold(bv, bi, c.v, c.i);
  }
  cv[tid] = bi < 0 ? -INFINITY : bv;
  const int n_max = static_cast<int>(block_sum<NT>(bi >= 0 ? 1ull : 0ull, s, sync));  // (its barriers publish cv)
  const float tau = N <= n_max ? kth_largest<NT>([&](int j) { return cv[j]; }, NT, N, s, sync) : -INFINITY;
  if (tid == 0) s.count = 0u;
  sync();
  for (int k0 = 0; k0 < m; k0 += NT) {
    const int k = k0 + tid;
    Cand c{0.f, -1};
    if (k < m) c = get(k);
    const bool take = c.i >= 0 && c.v >= tau;
    const unsigned ball = __ballot_sync(0xffffffffu, take);
    if (ball == 0u) continue;
    unsigned base = 0u;
    if (lane == 0) base = atomicAdd(&s.count, static_cast<unsigned>(__popc(ball)));
    base = __shfl_sync(0xffffffffu, base, 0);
    const int slot = static_cast<int>(base) + __popc(ball & ((1u << lane) - 1u));
    if (take && slot < cap) {
      cv[slot] = c.v;
      ci[slot] = c.i;
    }
  }
  sync();
  const int nc = static_cast<int>(s.count);
  if (tid < 32) {
    if (nc <= cap)
      warp_top_n([&](int k) { return Cand{cv[k], ci[k]}; }, nc, N, out_v, out_i);
    else
      warp_top_n(get, m, N, out_v, out_i);
  }
  sync();
}

// The record entry of one position (or the per-op outputs) by a block of NT threads, once m and lse_off are in
// ls and the top-N in ls.top_v / top_i: lp of `id` (logit read from l), then the top-N with their lp.  id outside
// [0, n): lp NaN.
__device__ __forceinline__ void write_entry(const float* l, int n, int id, int N, const LogprobScratch& ls,
                                            int32_t* out_id, float* out_lp, int32_t* top_ids, float* top_lp) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    if (out_id != nullptr) *out_id = id;
    *out_lp = (id >= 0 && id < n) ? logprob(__ldcg(l + id), ls.m, ls.lse_off) : __int_as_float(0x7fffffff);
  }
  if (tid < N) {
    const int i = ls.top_i[tid];
    top_ids[tid] = i;
    top_lp[tid] = i < 0 ? -INFINITY : logprob(ls.top_v[tid], ls.m, ls.lse_off);
  }
}

// The logprob rule over l[0..n) by one block of NT threads (the graph engine's argmax_advance_kernel and
// kllm_logprobs_f32): parts are the warps' contiguous ranges [w n / W, (w + 1) n / W).  Leaves m, lse_off and the
// top-N in ls (visible to the block on return).  scratch: logprob_scratch_bytes(NT) bytes, ls at its front.
template <int NT, class Sync>
__device__ __forceinline__ void logprobs_block(const float* l, int n, int N, unsigned char* scratch, int scratch_bytes,
                                               Sync sync) {
  constexpr int W = NT / 32;
  LogprobScratch& ls = *reinterpret_cast<LogprobScratch*>(scratch);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  sync();  // the scratch may still be read by a draw that just ended
  auto get = [&](int i) { return __ldcg(l + i); };
  const float2 p = warp_part(get, static_cast<int>(static_cast<long long>(warp) * n / W),
                             static_cast<int>(static_cast<long long>(warp + 1) * n / W));
  if (lane == 0) {
    ls.part_m[warp] = p.x;
    ls.part_s[warp] = p.y;
  }
  sync();
  if (warp == 0) {
    const float2 f = warp_fold_parts([&](int c) { return make_float2(ls.part_m[c], ls.part_s[c]); }, W);
    if (lane == 0) {
      ls.m = f.x;
      ls.lse_off = f.y;
    }
  }
  if (N > 0)
    top_n_block<NT>([&](int k) { return Cand{__ldcg(l + k), k}; }, n, N, scratch + kLogprobScratchBase,
                    scratch_bytes - kLogprobScratchBase, ls.top_v, ls.top_i, sync);
  else
    sync();
}

// Shared memory of a 1024-thread block's draw (up to 2048 candidates) and, after it, of its logprob routines
constexpr int kDrawScratchBytes = kDrawScratchBase + 2048 * 8;
static_assert(kDrawScratchBytes >= logprob_scratch_bytes(1024), "one scratch for the draw and the logprobs");

// The draw and record entry of one position by a block of 1024 threads (the graph engine's step and each position of
// kllm_decoder_verify): with step 0 on, the block first writes the adjusted logits to `penalized` (with pen's mark
// words) and draws from those; the raw logits are left as they are.  Then, with `record` and logprobs on, it writes
// the record entry at `pos` from the raw logits: of the drawn id, or of *target when target is set, which records
// even with logprobs off (kllm_decoder_score's targets).  Returns the drawn id (0 when the draw found none) in every
// thread.
__device__ __forceinline__ int draw_and_record(const float* logits, int n, const DrawSettings* cfg, PenaltyParams pen,
                                               float* penalized, const int32_t* hist, int pos, bool record,
                                               const int32_t* target, LogprobRecord rec) {
  __shared__ __align__(16) unsigned char scratch[kDrawScratchBytes];
  const float* l = logits;
  if (step0_active(pen)) {
    step0_history<1024>(logits, penalized, 0, n, pen, hist, pos, [] { __syncthreads(); });
    l = penalized;
  }
  const int bi = draw_block<1024>(l, n, cfg->sample, pos, nullptr, nullptr, 0, scratch, kDrawScratchBytes,
                                  [] { __syncthreads(); });
  const int id = bi < 0 ? 0 : bi;
  const int top_n = target != nullptr ? max(cfg->lp_top_n, 0) : cfg->lp_top_n;
  if (top_n >= 0 && record) {
    logprobs_block<1024>(logits, n, top_n, scratch, kDrawScratchBytes, [] { __syncthreads(); });
    const size_t row = static_cast<size_t>(pos) * kMaxTopLogprobs;
    write_entry(logits, n, target != nullptr ? *target : id, top_n, *reinterpret_cast<const LogprobScratch*>(scratch),
                rec.id + pos, rec.lp + pos, rec.top_ids + row, rec.top_lp + row);
  }
  return id;
}

}  // namespace sampling
}  // namespace kllm
