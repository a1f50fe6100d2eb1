// Persistent decode megakernel for sm_90a: the whole per-token forward of LLama2Model /
// Qwen2Model (kuiper/source/model/llama3.cpp:147-167, 600-745) in ONE cooperative launch that
// can run any number of consecutive positions.
//
// Why: at batch 1 the path is a 4-26 GB/token weight stream; with one launch per op (even 6
// fused launches per layer in a CUDA graph) every kernel boundary drains the HBM pipeline.
// Here one CTA per SM stays resident
// and a dedicated producer warp streams that CTA's share of EVERY weight matrix, in schedule
// order, through a ring of shared-memory stages with TMA bulk copies (cp.async.bulk ->
// UBLKCP) signalled on mbarriers.  Weights never depend on activations, so the producer runs
// ahead across every dependency of the token.
//
// Schedule per layer:  QKV(+bias) | attention(+RoPE) | Wo | W1,W3->SiLU*gate | W2 ; then
// classifier + greedy argmax.  RoPE moves into the attention phase so GEMV rows can be split
// evenly over all SMs.
//
// Consumers (kConsumerWarps = 8 warps): the rows of a ring stage are handed out as TASKS of
// up to four rows to one warp each, round-robin.  A task's rows share every load of the input vector, their
// dot-product chains interleave (ILP instead of occupancy), their totals are folded with "packed" shuffle trees
// (kllm_device.cuh) that do the additions of cub's tree only, and one lane per row runs the epilogues side by
// side.
//
// No local memory: the ring takes the whole unified L1, so a stack access is a round trip to L2.  The kernel
// parameters are __grid_constant__ (never copied to the stack), register buffers are always written in full
// (a conditionally written element forces the array into local memory), nothing indexes an array at run time.
// `cuobjdump -res-usage` / tools/sass_histogram.py show what is left.
//
// Hand-over between phases: every produced element is published as one 64-bit {tag, fp32} word and
// polled in place by the consuming phase -- no fences, flags or grid barriers; the residual-stream
// update after Wo and W2 is summed by the reader (x = x_old + sum over ranks, x_old living in the
// CTA's own shared memory), which under tensor parallelism makes the same stores, sent to every rank
// over NVLink peer mappings, the all-reduce.  Each token ends in exactly one grid barrier, after its
// last phase (the classifier, or the gather of the sharded classifier) and before the argmax fold;
// it is also what orders the producer's reads of the K/V rows the token wrote.
//
// Arithmetic is the same as the per-op kernels (gemv.cu / attention.cu / elementwise.cu): every
// dot product, reduction tree, softmax sum and value chain reproduces the reference CUDA
// kernels' floating-point order, so logits stay bit-identical to the reference's CUDA path.
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cfloat>
#include <cstdint>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/kllm_b200.h"
#include "kllm_device.cuh"
#include "kllm_host.h"
#include "kv_fp8.cuh"
#include "megakernel.h"

namespace kllm {
namespace mega {

// The phase bodies are written as functions but inlined: real calls make ptxas spill around them,
// and with the ring taking all of shared memory there is no L1 left -- a spill is an L2 round trip.
#define KLLM_MBAR_HINT_NS 20000u
#define KLLM_PHASE_CALL __forceinline__
#define KLLM_STAGE_CALL __noinline__  // once per phase, and their poll buffers would otherwise push the row loops' state out
constexpr int kMaxStages = 16;
// The consumer warps of every instantiation.  More consumer warps cap the registers of a thread below what the row
// loops need and ptxas spills on sm_90a (int8, 14 warps: 240 tok/s against 261 with 8 on an H100 SXM at 700 W).
constexpr int kConsumerWarps = 8;
constexpr int kConsumerThreads = kConsumerWarps * 32;
constexpr int kSoftmaxThreads = 256;  // mha_kernel.cu:112-127 launches 256 threads per head
constexpr int kNormThreads = 128;     // rmsnorm_kernel.cu:58-77 launches 128 threads
constexpr long long kSpinLimit = 120000000000LL;  // ~1 minute of SM clocks: a lost peer becomes a trap

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* b, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
// try_wait suspends the warp in hardware until the phase completes or the time hint (ns) runs out:
// with a generous hint a waiting warp sleeps instead of re-issuing the probe -- waiting warps
// otherwise compete for issue slots with the warps that are computing on the same scheduler
// (ncu, r02f: SYNCS + BRA + YIELD of the spin loops were a quarter of all executed instructions).
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  asm volatile(
      "{\n .reg .pred p;\n WAIT_%=:\n"
      " mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      " @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" ::"r"(smem_u32(b)),
      "r"(parity), "r"(KLLM_MBAR_HINT_NS)
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n"
      " mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
      " selp.u32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(smem_u32(b)), "r"(parity), "r"(KLLM_MBAR_HINT_NS)
      : "memory");
  return ok != 0;
}
// The producer's wait on a stage's `empty` barrier in a stoppable run: a stopped CTA's consumers never free
// the slot, so the wait gives up once *stop is set.  Warp-uniform: true (stop, issue nothing) if any lane saw
// the flag; a copy is issued only when every lane saw the slot free.
__device__ __forceinline__ bool mbar_wait_or_stop(uint64_t* b, uint32_t parity, const volatile int* stop) {
  bool stopped = false;
  while (!mbar_try_wait(b, parity)) {
    if (*stop) {
      stopped = true;
      break;
    }
  }
  return __any_sync(0xffffffffu, stopped);
}
__device__ __forceinline__ void st_release_sys(int32_t* p, int32_t v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar,
                                         uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// 64-bit {tag, value} words of the tagged exchange: single-copy atomic, so value and tag travel
// together and no fence or flag is needed between a writer on one GPU and a reader on another.
__device__ __forceinline__ unsigned long long tagged_word(float v, unsigned tag) {
  return (static_cast<unsigned long long>(tag) << 32) | __float_as_uint(v);
}
__device__ __forceinline__ void st_tagged(unsigned long long* p, float v, unsigned tag) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(tagged_word(v, tag)) : "memory");
}
__device__ __forceinline__ void ld_tagged2(const unsigned long long* p, unsigned long long& a,
                                           unsigned long long& b) {
  asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
// local (same GPU) flavour of the tagged words
__device__ __forceinline__ void st_tagged_gpu(unsigned long long* p, float v, unsigned tag) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(tagged_word(v, tag)) : "memory");
}
__device__ __forceinline__ void st_tagged2_gpu(unsigned long long* p, float v0, float v1, unsigned tag) {  // 16-byte aligned
  asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(tagged_word(v0, tag)), "l"(tagged_word(v1, tag))
               : "memory");
}
__device__ __forceinline__ unsigned long long ld_tagged_gpu(const unsigned long long* p) {
  unsigned long long w;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
  return w;
}
__device__ __forceinline__ void ld_tagged2_gpu(const unsigned long long* p, unsigned long long& a,
                                               unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ unsigned tag_of(unsigned long long w) { return static_cast<unsigned>(w >> 32); }
__device__ __forceinline__ float val_of(unsigned long long w) { return __uint_as_float(static_cast<unsigned>(w)); }

// A polled word may carry an OLDER tag (its producer is still on its way) but never a NEWER one:
// the slot-reuse argument (megakernel.h) says nobody publishes use n+1 of a word before everybody
// consumed use n.  A newer tag is therefore a protocol error and traps at once; a word that never
// turns up becomes a trap after a bounded spin, not a hang.
__device__ __noinline__ void poll_failed(unsigned seen, unsigned want, long long t_start, int what) {
  const char* name = what == 0 ? "hand-off word" : (what == 1 ? "residual exchange" : "phase input");
  if (static_cast<int>(seen - want) > 0) {
    printf("kllm mega: cta %d thread %d: %s carries tag %u, newer than the awaited %u (protocol error)\n",
           blockIdx.x, threadIdx.x, name, seen, want);
    __trap();
  }
  if (clock64() - t_start > kSpinLimit) {
    printf("kllm mega: cta %d thread %d timed out on %s tag %u (last seen %u)\n", blockIdx.x, threadIdx.x,
           name, want, seen);
    __trap();
  }
}
__device__ __forceinline__ unsigned long long ld_tagged_sys(const unsigned long long* p) {
  unsigned long long w;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
  return w;
}
// spin until the word (written by any rank) carries `tag`
__device__ __forceinline__ float poll_tagged_sys(const unsigned long long* p, unsigned tag) {
  unsigned long long w = ld_tagged_sys(p);
  if (tag_of(w) != tag) {
    const long long t0 = clock64();
    do {
      poll_failed(tag_of(w), tag, t0, 1);
      w = ld_tagged_sys(p);
    } while (tag_of(w) != tag);
  }
  return val_of(w);
}
// spin until the word carries `tag`
__device__ __forceinline__ float poll_tagged(const unsigned long long* p, unsigned tag) {
  unsigned long long w = ld_tagged_gpu(p);
  if (tag_of(w) != tag) {
    const long long t0 = clock64();
    do {
      poll_failed(tag_of(w), tag, t0, 0);
      w = ld_tagged_gpu(p);
    } while (tag_of(w) != tag);
  }
  return val_of(w);
}
__device__ __forceinline__ void consumer_sync() {
  asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

struct Pipe {
  int slot;
  uint32_t parity;
  __device__ __forceinline__ void advance(int stages) {
    if (++slot == stages) {
      slot = 0;
      parity ^= 1u;
    }
  }
};

// Static shared memory (namespace scope, so the phase functions address it with immediates instead of
// pointers held in registers).  The ring leaves only a few KB of L1, so everything the inner loops
// touch lives in shared memory or registers: the schedule entries the consumers and the ring producer
// are working on (usually two different phases), the barriers and the reduction scratch.
__shared__ uint64_t g_full_bar[kMaxStages];
__shared__ uint64_t g_empty_bar[kMaxStages];
__shared__ float g_s_warp[kConsumerWarps];
__shared__ float g_s_argv[kConsumerWarps];
__shared__ int g_s_argi[kConsumerWarps];
__shared__ float g_s_bcast;
// Stoppable runs (Params::stop_ids): the consumers set g_stop once the token's id is a stop id; the producer
// then stops issuing and publishes where its ring position ended, 1 + (slot << 1 | parity), in g_prod_end
// (0: still running).  The consumers drain every fill up to that position before the CTA exits.
__shared__ volatile int g_stop;
__shared__ volatile unsigned g_prod_end;
__shared__ Phase g_ph_cons;
__shared__ Phase g_ph_prod;
extern __shared__ __align__(128) unsigned char smem[];
// per-thread state the phase functions hand back to the kernel loop
struct Carry {
  Pipe pipe;
  float best_v;
  int best_i;
};

// Grid barrier over the consumer threads of all CTAs.  Monotonic counter, wrap-safe compare.
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned& target, unsigned grid) {
  consumer_sync();
  target += grid;
  if (threadIdx.x == 0) {
    red_release_add(counter, 1u);
    while (static_cast<int>(ld_acquire_u32(counter) - target) < 0) {
    }
  }
  consumer_sync();
}

// ---- unit -> (segment, row) ------------------------------------------------------------------
struct RowRef {
  int seg;
  int row;
};
__device__ __forceinline__ RowRef resolve_row(const Phase& ph, int unit, int sub) {
  if (ph.swiglu) return RowRef{sub, unit};
  int seg = 0, row = unit;
  if (ph.n_seg > 1 && row >= ph.seg[0].rows) {
    row -= ph.seg[0].rows;
    seg = 1;
    if (ph.n_seg > 2 && row >= ph.seg[1].rows) {
      row -= ph.seg[1].rows;
      seg = 2;
    }
  }
  return RowRef{seg, row};
}

// Row j of a ring stage that starts at unit u and holds n units, in STAGE ORDER.  SwiGLU stages
// keep their w1 rows first and their w3 rows after them, so that each half -- like any run of
// consecutive rows of one matrix -- is ONE contiguous span of the checkpoint and one bulk copy.
__device__ __forceinline__ RowRef stage_row(const Phase& ph, int u, int n, int j) {
  if (ph.swiglu) return j < n ? RowRef{0, u + j} : RowRef{1, u + j - n};
  return resolve_row(ph, u + j, 0);
}
// Lane j (< nrows) holds row j of the stage: returns the length of the run of consecutive rows
// of one matrix that STARTS at this lane (0 for lanes inside a run).
__device__ __forceinline__ int run_length(const RowRef& rr, int lane, int nrows) {
  const int pseg = __shfl_up_sync(kFull, rr.seg, 1);
  const int prow = __shfl_up_sync(kFull, rr.row, 1);
  const bool head = lane < nrows && (lane == 0 || rr.seg != pseg || rr.row != prow + 1);
  const unsigned heads = __ballot_sync(kFull, head);
  if (!head) return 0;
  const unsigned later = heads & ~((2u << lane) - 1u);
  return (later ? __ffs(later) - 1 : nrows) - lane;
}

// ---- exact-order accumulation from shared memory ----------------------------------------------
// The row loops address shared memory by 32-bit shared-window addresses through explicit
// ld.shared: behind the call boundary of dot_rows the compiler no longer knows the pointers are
// shared memory (it would emit generic loads), and `volatile` keeps the loads in program order --
// a batch of loads first, then the math that consumes them.
__device__ __forceinline__ float4 lds_f4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ float lds_f32(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
  return v;
}
// bf16 KV cache: an element widened exactly to fp32 (the bf16 bits are the float's upper half)
__device__ __forceinline__ float lds_bf16(uint32_t a) {
  unsigned short v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a));
  return __uint_as_float(static_cast<uint32_t>(v) << 16);
}
// fp8 KV cache: value(code) of the e4m3 code at a, exact
__device__ __forceinline__ float lds_e4m3(uint32_t a) {
  unsigned short v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=h"(v) : "r"(a));
  return e4m3_value(static_cast<uint8_t>(v));
}
// the two bf16 elements of a 32-bit word (held as a float's bits): element 2i in the low half, 2i + 1 in the high
__device__ __forceinline__ float bf16_lo(float w) { return __uint_as_float(__float_as_uint(w) << 16); }
__device__ __forceinline__ float bf16_hi(float w) { return __uint_as_float(__float_as_uint(w) & 0xffff0000u); }

// fp32 and bf16 rows: virtual thread (lane + 32 j) owns packs base + 32 j + lane (matmul_kernel.cu:27-35).  A pack
// is four weights, 4 * weight_bytes(F) bytes: one 16-byte load of fp32, or one 8-byte load of bf16 (a warp reads 256
// consecutive bytes: no bank conflicts) widened exactly to fp32, so every dot4 and addition is the fp32 kernel's over
// the widened weights.  The NR rows of a task share each load of x; per batch (two 32-pack columns) 2 x loads and
// 2 NR weight loads are issued before the 2 NR independent dot4 chains.
__device__ __forceinline__ float4 lds_bf16x4(uint32_t a) {
  uint32_t lo, hi;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(lo), "=r"(hi) : "r"(a));
  return widen_bf16x4(lo, hi);
}
template <WeightFormat F>
__device__ __forceinline__ float4 lds_pack(uint32_t a) {
  if constexpr (F == WeightFormat::kBf16)
    return lds_bf16x4(a);
  else
    return lds_f4(a);
}
template <int NR, WeightFormat F>
__device__ __forceinline__ void accum_packs(const uint32_t (&w)[NR], uint32_t x, int n_packs, int lane,
                                            float (&acc)[NR][4]) {
  constexpr int PB = 4 * weight_bytes(F);  // bytes per pack
  // Full 128-pack blocks run branch-free with all 4 * (1 + NR) shared loads issued before the math
  // (two blocks in flight), so the four independent chains per row overlap the LDS latency.
  const int full = n_packs & ~127;
  uint32_t xp = x + lane * 16;
  uint32_t wp[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) wp[r] = w[r] + lane * PB;
#pragma unroll 2
  for (int base = 0; base < full; base += 128) {
    float4 xv[4];
    float4 wv[NR][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) xv[j] = lds_f4(xp + 512 * j);
#pragma unroll
    for (int r = 0; r < NR; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) wv[r][j] = lds_pack<F>(wp[r] + 32 * PB * j);
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int r = 0; r < NR; ++r) acc[r][j] = __fadd_rn(dot4_ref(xv[j], wv[r][j]), acc[r][j]);
    xp += 2048;
#pragma unroll
    for (int r = 0; r < NR; ++r) wp[r] += 128 * PB;
  }
  if (full < n_packs) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (full + 32 * j + lane < n_packs) {
        const float4 xv = lds_f4(xp + 512 * j);
#pragma unroll
        for (int r = 0; r < NR; ++r) acc[r][j] = __fadd_rn(dot4_ref(xv, lds_pack<F>(wp[r] + 32 * PB * j)), acc[r][j]);
      }
    }
  }
}

// int8, group size 64 (export.py --version 3): virtual thread (4 lane + e) owns elements
// 128 k + 4 lane + e (matmul_kernel.cu:70-74), so the lane's four bytes of chunk k sit in group
// 2 k + (lane >> 4) of the row: the scale address just steps by two floats.  Per element the
// reference's fma(x * scale, float(w), acc) -- PRMT + FADD (exact int8 -> fp32) + FMUL + FFMA;
// everything else (one 4-byte weight load and one scale load per row, one 16-byte x load per chunk,
// the xor that prepares the byte permutes) is shared by four elements or by the NR rows.  Chunk
// k + 1 is loaded while chunk k is computed.
// `sc[r]`: the row's staged scales (rows start on a group boundary -- checked on the host).
template <int NR>
__device__ __forceinline__ void accum_w8_g64(const uint32_t (&w)[NR], const uint32_t (&sc)[NR], uint32_t x,
                                             int M, int lane, float (&acc)[NR][4]) {
  const int chunks = M >> 7;
  const bool tail = (chunks << 7) + (lane << 2) < M;  // M % 128 != 0: a last, partial chunk
  const int total = chunks + (tail ? 1 : 0);
  if (total == 0) return;
  uint32_t xp = x + lane * 16;
  uint32_t wp[NR], sp[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    wp[r] = w[r] + lane * 4;
    sp[r] = sc[r] + (lane >> 4) * 4;
  }
  float4 xv = lds_f4(xp);
  uint32_t packed[NR];
  float s[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    packed[r] = lds_u32(wp[r]);
    s[r] = lds_f32(sp[r]);
  }
#pragma unroll 2
  for (int k = 0; k < total; ++k) {
    if (k + 1 < total) {  // uniform per virtual-thread quad: lanes past a partial tail chunk have total == chunks
      xp += 512;
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        wp[r] += 128;
        sp[r] += 8;
      }
    }
    const float4 xn = lds_f4(xp);  // last iteration: re-reads its own chunk (harmless)
    uint32_t pn[NR];
    float sn[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      pn[r] = lds_u32(wp[r]);
      sn[r] = lds_f32(sp[r]);
    }
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      float wf[4];
      int8x4_to_float(packed[r], wf);
      acc[r][0] = __fmaf_rn(__fmul_rn(xv.x, s[r]), wf[0], acc[r][0]);
      acc[r][1] = __fmaf_rn(__fmul_rn(xv.y, s[r]), wf[1], acc[r][1]);
      acc[r][2] = __fmaf_rn(__fmul_rn(xv.z, s[r]), wf[2], acc[r][2]);
      acc[r][3] = __fmaf_rn(__fmul_rn(xv.w, s[r]), wf[3], acc[r][3]);
    }
    xv = xn;
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      packed[r] = pn[r];
      s[r] = sn[r];
    }
  }
}

// int8, any other group size (multiple of 4): the group index is computed per chunk.
template <int NR>
__device__ __forceinline__ void accum_w8_any(const uint32_t (&w)[NR], const uint32_t (&sc)[NR], uint32_t x,
                                             int M, int group_shift, int group_size, int lane,
                                             float (&acc)[NR][4]) {
  const int full_chunks = M >> 7;
  auto one = [&](int k) {
    const int i = (k << 7) + (lane << 2);
    const float4 xv = lds_f4(x + i * 4);
    const int g = group_shift >= 0 ? (i >> group_shift) : (i / group_size);
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      const uint32_t packed = lds_u32(w[r] + i);
      const float s = lds_f32(sc[r] + g * 4);
      float wf[4];
      int8x4_to_float(packed, wf);
      acc[r][0] = __fmaf_rn(__fmul_rn(xv.x, s), wf[0], acc[r][0]);
      acc[r][1] = __fmaf_rn(__fmul_rn(xv.y, s), wf[1], acc[r][1]);
      acc[r][2] = __fmaf_rn(__fmul_rn(xv.z, s), wf[2], acc[r][2]);
      acc[r][3] = __fmaf_rn(__fmul_rn(xv.w, s), wf[3], acc[r][3]);
    }
  };
#pragma unroll 2
  for (int k = 0; k < full_chunks; ++k) one(k);
  if ((full_chunks << 7) + (lane << 2) < M) one(full_chunks);
}

// ---- int8 weights x fixed-point activations on the integer dot-product unit (TOLERANCED) ---------
// The exact int8 loop above is bound by instruction issue: four instructions per weight byte
// (PRMT + FADD to convert, FMUL by the group scale, FFMA), ~21 warp instructions per 128 weight
// bytes against ~5.6 bytes per clock per scheduler that HBM can deliver.  The fast mode turns the
// activations of each 64-element group into 24-bit fixed point once per phase --
//     x_i ~= step_g * q_i,  q_i = round(x_i / step_g),  step_g = max|x in group| / 2^22,
// q_i split into three balanced base-256 digits l2 l1 l0 (int8 each) -- and then needs ONE dp4a per
// 4 weights and digit: sum_i w_i x_i = s_g * step_g * (65536 D2 + 256 D1 + D0), D_k = sum_i w_i l_k,i
// exact in int32.  ~6 warp instructions per 128 weight bytes.  The group scale s_g and the int8
// weights enter exactly as in the reference (dequantised weight = q * s, export.py:60-67); only x is
// rounded, to within 2^-22 of its group maximum (half a step, 2^-23, plus what the rounded reciprocal
// `inv` adds: tests/test_decode_model.py pins the bound) -- the order of fp32 rounding of the products
// themselves.  Logits agree with the exact mode to ~1e-6 relative (tests: <= 1e-4 absolute, same
// greedy id wherever the top-2 margin exceeds 2e-4), not bit for bit.
__device__ __forceinline__ uint4 lds_u4(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ int dp4a4(const uint4& w, const uint4& l) {
  int d = __dp4a(static_cast<int>(w.x), static_cast<int>(l.x), 0);
  d = __dp4a(static_cast<int>(w.y), static_cast<int>(l.y), d);
  d = __dp4a(static_cast<int>(w.z), static_cast<int>(l.z), d);
  return __dp4a(static_cast<int>(w.w), static_cast<int>(l.w), d);
}
// exact int32 -> fp32 for |d| < 2^22 without the slow conversion pipe: 1.5 * 2^23 + d is exact
__device__ __forceinline__ float small_int_to_float(int d) {
  return __fsub_rn(__int_as_float(0x4B400000 + d), 12582912.0f);
}
// In-place layout (fast mode): the 256 bytes that held the fp32 values of 64-element group g hold four
// 64-byte regions -- the three digit planes of the group and its step.  Digit plane k sits in region
// (k + (g & 1)) & 3, the step in region (3 + (g & 1)) & 3: alternating the region order between even
// and odd groups makes the 32 lanes of a 128-bit load (8 groups x 4 quarters) hit all 8 distinct
// 16-byte bank slots, 4 lanes each -- the minimum of 4 wavefronts.  Quarter q (16 elements) of a
// plane is the 16-byte chunk q of its region.
template <int NR>
__device__ __forceinline__ void accum_w8_dp4a(const uint32_t (&w)[NR], const uint32_t (&sc)[NR], uint32_t x, int M,
                                              int lane, float (&acc)[NR]) {
  // lane owns 16 consecutive elements per step of 512: group = 8 * step + lane / 4, quarter = lane % 4
  const uint32_t odd = (lane >> 2) & 1u;
  const uint32_t gq = x + (lane >> 2) * 256 + (lane & 3) * 16;
  const uint32_t l0 = gq + ((0u + odd) & 3u) * 64, l1 = gq + ((1u + odd) & 3u) * 64, l2 = gq + ((2u + odd) & 3u) * 64;
  const uint32_t xsp = x + (lane >> 2) * 256 + ((3u + odd) & 3u) * 64;
  uint32_t wp[NR], sp[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    wp[r] = w[r] + lane * 16;
    sp[r] = sc[r] + (lane >> 2) * 4;
  }
  const int steps = (M + 511) >> 9;
#pragma unroll 2
  for (int it = 0; it < steps; ++it) {
    if (it * 512 + lane * 16 < M) {  // M % 512 != 0: the last step covers part of the lanes (M % 64 == 0)
      const uint4 a0 = lds_u4(l0 + it * 2048), a1 = lds_u4(l1 + it * 2048), a2 = lds_u4(l2 + it * 2048);
      const float xstep = lds_f32(xsp + it * 2048);
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        const uint4 wv = lds_u4(wp[r] + it * 512);
        const float ws = lds_f32(sp[r] + it * 32);
        const float c0 = small_int_to_float(dp4a4(wv, a0));
        const float c1 = small_int_to_float(dp4a4(wv, a1));
        const float c2 = small_int_to_float(dp4a4(wv, a2));
        const float f = __fmaf_rn(c2, 65536.0f, __fmaf_rn(c1, 256.0f, c0));
        acc[r] = __fmaf_rn(f, __fmul_rn(xstep, ws), acc[r]);
      }
    }
  }
}

// The phase's input vector (fp32, M floats at xs, M % 64 == 0) -> digit planes + step per group, in
// place (layout above).  Four adjacent lanes share a group: each reads its 16 values, the group
// maximum is folded with two shuffles, and after a warp-level sync (all four have read) each lane
// overwrites its quarter -- no CTA barrier, no values parked in registers.
__device__ __noinline__ void quantize_input_inplace(float* xs, int M, int tid) {
  const int quarters = M >> 4;
  for (int base = 0; base < quarters; base += kConsumerThreads) {  // whole warps: groups never straddle one
    const int qg = base + tid;
    const bool on = qg < quarters;
    // lanes past the end read the last quarter again (their group is entirely past the end: M % 64 == 0),
    // so v[] is always written and stays in registers instead of local memory
    float4 v[4];
    float gmax = 0.f;
    {
      const float4* g4 = reinterpret_cast<const float4*>(xs) + min(qg, quarters - 1) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        v[j] = g4[j];
        gmax = fmaxf(gmax, fmaxf(fmaxf(fabsf(v[j].x), fabsf(v[j].y)), fmaxf(fabsf(v[j].z), fabsf(v[j].w))));
      }
    }
    gmax = fmaxf(gmax, __shfl_xor_sync(kFull, gmax, 1));
    gmax = fmaxf(gmax, __shfl_xor_sync(kFull, gmax, 2));  // also orders: every lane of the group has read
    const float step = gmax * (1.0f / 4194304.0f);      // 2^-22
    const float inv = gmax > 0.f ? 4194304.0f / gmax : 0.f;
    __syncwarp();
    if (on) {
      const int g = qg >> 2, q = qg & 3;
      const unsigned odd = g & 1;
      unsigned char* gb = reinterpret_cast<unsigned char*>(xs) + g * 256 + q * 16;
      uint32_t* o0 = reinterpret_cast<uint32_t*>(gb + ((0u + odd) & 3u) * 64);
      uint32_t* o1 = reinterpret_cast<uint32_t*>(gb + ((1u + odd) & 3u) * 64);
      uint32_t* o2 = reinterpret_cast<uint32_t*>(gb + ((2u + odd) & 3u) * 64);
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // 4 elements -> one word of each digit plane, written at once
        const float e[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
        uint32_t p0 = 0, p1 = 0, p2 = 0;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int qv = __float2int_rn(e[b] * inv);  // |qv| <= 2^22
          const int a0 = ((qv + 128) & 255) - 128;    // balanced digits: qv = 65536 a2 + 256 a1 + a0
          const int q1 = (qv - a0) >> 8;
          const int a1 = ((q1 + 128) & 255) - 128;
          const int a2 = (q1 - a1) >> 8;
          p0 |= static_cast<uint32_t>(a0 & 255) << (8 * b);
          p1 |= static_cast<uint32_t>(a1 & 255) << (8 * b);
          p2 |= static_cast<uint32_t>(a2 & 255) << (8 * b);
        }
        o0[j] = p0, o1[j] = p1, o2[j] = p2;
      }
      if (q == 0) *reinterpret_cast<float*>(gb + ((3u + odd) & 3u) * 64) = step;
    }
  }
  consumer_sync();
}

// Dot products of the NR rows of a task (shared-window addresses of the rows and of their int8
// scales); every lane gets every total.  Deliberately NOT inlined: as part of the megakernel's one
// big function the row loops inherit its register pressure and ptxas then serialises every
// shared-memory load with its dependent math; as a function of their own they keep a batch of loads
// in flight.
struct Rows4 {
  uint32_t a[4];
};
template <int NR, WeightFormat F>
__device__ __forceinline__ float4 dot_rows(Rows4 rows, Rows4 scales, uint32_t x, int M, int group_size,
                                           int group_shift, int lane, bool fast = false) {
  float acc[NR][4];
#pragma unroll
  for (int r = 0; r < NR; ++r)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[r][j] = 0.f;
  float d[4] = {0.f, 0.f, 0.f, 0.f};
  uint32_t w[NR], sc[NR];
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    w[r] = rows.a[r];
    sc[r] = scales.a[r];
  }
  if constexpr (F == WeightFormat::kInt8) {
    if (fast) {  // fixed-point activations x int8 weights on dp4a (toleranced mode; group size 64)
      float a1[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) a1[r] = 0.f;
      accum_w8_dp4a<NR>(w, sc, x, M, lane, a1);
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        float v = a1[r];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
        d[r] = v;
      }
      return make_float4(d[0], d[1], d[2], d[3]);
    }
    if (group_size == 64)
      accum_w8_g64<NR>(w, sc, x, M, lane, acc);
    else
      accum_w8_any<NR>(w, sc, x, M, group_shift, group_size, lane, acc);
#pragma unroll
    for (int r = 0; r < NR; ++r) d[r] = block128_sum_quad_packed(acc[r]);
  } else {
    accum_packs<NR, F>(w, x, M >> 2, lane, acc);
#pragma unroll
    for (int r = 0; r < NR; ++r) d[r] = block128_sum_vt_packed(acc[r], lane);
  }
  return make_float4(d[0], d[1], d[2], d[3]);
}

struct ArgBest {
  float v;
  int i;
};
__device__ __forceinline__ void arg_fold(ArgBest& a, float ov, int oi) {
  if (oi >= 0 && (a.i < 0 || ov > a.v || (ov == a.v && oi < a.i))) {
    a.v = ov;
    a.i = oi;
  }
}

// ---- staging of a tagged input vector ------------------------------------------------------------
// Residual exchange (tp_in): x = x_old + (p_0 + ... + p_{W-1}); the partials of every rank (this
// one included) arrive as tagged words in this rank's exchange area and are polled in place; x_old
// is the CTA's own copy of the residual stream in shared memory (xres), updated here.  Thread t
// handles packs t, t + NT, ...; UP packs x W ranks x 2 loads are in flight per poll round.
// With W == 1 and FOLD the rmsnorm sum of squares is accumulated in the same pass by the
// kNormThreads threads that own the reference's chains (rmsnorm_kernel.cu:19-32).
template <int W, int UP, bool FOLD>
__device__ KLLM_STAGE_CALL float stage_exchange(const unsigned long long* area, int tp_stride, unsigned tag, int n4,
                                                int t, int NT, float4* xs4, float4* xres4) {
  float ssq = 0.f;
  const long long t_start = clock64();
  for (int pb = t; pb < n4; pb += NT * UP) {
    // Every slot of the batch loads SOMETHING (slots past the end re-read the last pack): a buffer
    // with conditionally written elements is kept in local memory by the compiler, and with the ring
    // taking the whole unified L1 a local-memory access is an L2 round trip per poll round.
    unsigned long long wd[UP][W][4];
    bool ok;
    unsigned seen = tag;
    do {
      ok = true;
#pragma unroll
      for (int k = 0; k < UP; ++k) {
        const int p = min(pb + k * NT, n4 - 1);
#pragma unroll
        for (int r = 0; r < W; ++r) {
          const unsigned long long* row = area + static_cast<size_t>(r) * tp_stride + 4 * p;
          if (W == 1) {
            ld_tagged2_gpu(row, wd[k][r][0], wd[k][r][1]);
            ld_tagged2_gpu(row + 2, wd[k][r][2], wd[k][r][3]);
          } else {
            ld_tagged2(row, wd[k][r][0], wd[k][r][1]);
            ld_tagged2(row + 2, wd[k][r][2], wd[k][r][3]);
          }
        }
      }
#pragma unroll
      for (int k = 0; k < UP; ++k)
#pragma unroll
        for (int r = 0; r < W; ++r)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (tag_of(wd[k][r][e]) != tag) {
              ok = false;
              seen = tag_of(wd[k][r][e]);
            }
      if (!ok) poll_failed(seen, tag, t_start, 1);
    } while (!ok);
#pragma unroll
    for (int k = 0; k < UP; ++k) {
      const int p = pb + k * NT;
      if (p < n4) {
        float s[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          s[e] = val_of(wd[k][0][e]);
#pragma unroll
          for (int r = 1; r < W; ++r) s[e] = __fadd_rn(s[e], val_of(wd[k][r][e]));  // rank order
        }
        float4 x = xres4[p];
        x.x = __fadd_rn(x.x, s[0]);  // llama3.cpp:683,719: x + out
        x.y = __fadd_rn(x.y, s[1]);
        x.z = __fadd_rn(x.z, s[2]);
        x.w = __fadd_rn(x.w, s[3]);
        xres4[p] = x;
        xs4[p] = x;
        if (FOLD) {
          ssq = __fmaf_rn(x.x, x.x, ssq);
          ssq = __fmaf_rn(x.y, x.y, ssq);
          ssq = __fmaf_rn(x.z, x.z, ssq);
          ssq = __fmaf_rn(x.w, x.w, ssq);
        }
      }
    }
  }
  return ssq;
}

// Local hand-off (tag_in): the previous phase's output vector, polled in place.
template <int UP>
__device__ __forceinline__ void stage_handoff_inline(const unsigned long long* src, unsigned tag, int n4, int t, int NT,
                                                     float4* xs4) {
  const long long t_start = clock64();
  for (int pb = t; pb < n4; pb += NT * UP) {
    unsigned long long wd[UP][4];  // every slot loads (clamped index): keeps the buffer in registers, see stage_exchange
    bool ok;
    unsigned seen = tag;
    do {
      ok = true;
#pragma unroll
      for (int k = 0; k < UP; ++k) {
        const int p = min(pb + k * NT, n4 - 1);
        ld_tagged2_gpu(src + 4 * p, wd[k][0], wd[k][1]);
        ld_tagged2_gpu(src + 4 * p + 2, wd[k][2], wd[k][3]);
      }
#pragma unroll
      for (int k = 0; k < UP; ++k)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (tag_of(wd[k][e]) != tag) {
            ok = false;
            seen = tag_of(wd[k][e]);
          }
      if (!ok) poll_failed(seen, tag, t_start, 2);
    } while (!ok);
#pragma unroll
    for (int k = 0; k < UP; ++k) {
      const int p = pb + k * NT;
      if (p < n4) xs4[p] = make_float4(val_of(wd[k][0]), val_of(wd[k][1]), val_of(wd[k][2]), val_of(wd[k][3]));
    }
  }
}
template <int UP>
__device__ KLLM_STAGE_CALL void stage_handoff(const unsigned long long* src, unsigned tag, int n4, int t, int NT,
                                              float4* xs4) {
  stage_handoff_inline<UP>(src, tag, n4, t, NT, xs4);
}

// ---- inputs of an attention CTA: q (this head), raw k and v (its kv head) of the current position ------------
// Thread i < hs/2 needs its pair of q (and, in the CTA that handles the new key row, of k); thread d < hs the
// value element d.  With tagged hand-offs these are up to five words per thread; polled one after the other
// (each poll a spin loop of its own) they cost five dependent L2 round trips at the head of the layer's
// critical path -- here all of a thread's words are in flight together and re-read together until every tag is
// current.  Slots a thread does not need alias a word it does need.
struct AttnIn {
  float q0, q1, k0, k1, v;
};
__device__ __forceinline__ AttnIn poll_attention_inputs(const unsigned long long* pq0, const unsigned long long* pq1,
                                                        const unsigned long long* pk0, const unsigned long long* pk1,
                                                        const unsigned long long* pv, unsigned tag) {
  unsigned long long w[5];
  w[0] = ld_tagged_gpu(pq0), w[1] = ld_tagged_gpu(pq1), w[2] = ld_tagged_gpu(pk0), w[3] = ld_tagged_gpu(pk1);
  w[4] = ld_tagged_gpu(pv);
  // (no dynamic index into w[]: that would put the buffer into local memory)
  unsigned seen = tag;
  auto stale = [&]() -> bool {
    bool bad = false;
#pragma unroll
    for (int i = 0; i < 5; ++i)
      if (tag_of(w[i]) != tag) bad = true, seen = tag_of(w[i]);
    return bad;
  };
  if (stale()) {
    const long long t0 = clock64();
    do {
      poll_failed(seen, tag, t0, 0);
      w[0] = ld_tagged_gpu(pq0), w[1] = ld_tagged_gpu(pq1), w[2] = ld_tagged_gpu(pk0), w[3] = ld_tagged_gpu(pk1);
      w[4] = ld_tagged_gpu(pv);
    } while (stale());
  }
  return AttnIn{val_of(w[0]), val_of(w[1]), val_of(w[2]), val_of(w[3]), val_of(w[4])};
}

// RoPE on q (this head) and -- with_k -- on the new key row (rope_kernel.cu as compiled, elementwise.cu); the
// rotated key goes to k_s and, by one CTA per kv head, into the cache row of `pos` (rounded to bf16 with
// the bf16 KV cache, encoded at its layer's and kv head's scale with the fp8 one: KV, a kllm_decoder_desc::kv_cache
// value).  Returns this thread's element of the value row (with_v, tid < hs), else 0.
template <int KV = KLLM_KV_F32>
__device__ __forceinline__ float attention_inputs(const Params& P, const Phase& ph, int head, int kvh, int pos, unsigned tag_in,
                                                  bool with_k, bool with_v, float* q_s, float* k_s, size_t head_block) {
  const int tid = threadIdx.x;
  const int hs = P.head_size, seq_len = P.seq_len;
  const bool need_q = tid < hs / 2, need_k = need_q && with_k, need_v = with_v && tid < hs;
  if (!need_q && !need_v) return 0.f;
  int i0, i1;
  if (P.flavour == KLLM_FLAVOUR_LLAMA2) {
    i0 = 2 * tid, i1 = 2 * tid + 1;
  } else {
    i0 = tid, i1 = tid + hs / 2;
  }
  const unsigned long long* pv = ph.tv + kvh * hs + tid;
  const unsigned long long* pq0 = ph.tq + head * hs + i0;
  const unsigned long long* pq1 = ph.tq + head * hs + i1;
  const unsigned long long* any = need_q ? pq0 : pv;  // a word this thread waits for anyway
  const AttnIn in = poll_attention_inputs(need_q ? pq0 : any, need_q ? pq1 : any, need_k ? ph.tk + kvh * hs + i0 : any,
                                          need_k ? ph.tk + kvh * hs + i1 : any, need_v ? pv : any, tag_in);
  if (need_q) {
    const int ci = 2 * tid;
    const float fci = P.sin_cache[static_cast<size_t>(pos) * hs + ci];
    const float fcr = P.cos_cache[static_cast<size_t>(pos) * hs + ci];
    q_s[i0] = __fmaf_rn(fcr, in.q0, -__fmul_rn(fci, in.q1));
    q_s[i1] = __fmaf_rn(fci, in.q0, __fmul_rn(fcr, in.q1));
    if (need_k) {
      const float r0 = __fmaf_rn(fcr, in.k0, -__fmul_rn(fci, in.k1));
      const float r1 = __fmaf_rn(fci, in.k0, __fmul_rn(fcr, in.k1));
      k_s[i0] = r0;
      k_s[i1] = r1;
      if (head % P.kv_mul == 0) {  // one writer per kv head stores the rotated key
        if constexpr (KV == KLLM_KV_FP8) {
          uint8_t* kcache = reinterpret_cast<uint8_t*>(P.key_cache) + head_block;
          const float inv = P.kv_inv_k[ph.layer * (P.kv_dim / hs) + kvh];
          kcache[(static_cast<size_t>(i0 >> 4) * seq_len + pos) * 16 + (i0 & 15)] = e4m3_encode(r0, inv);
          kcache[(static_cast<size_t>(i1 >> 4) * seq_len + pos) * 16 + (i1 & 15)] = e4m3_encode(r1, inv);
        } else if constexpr (KV == KLLM_KV_BF16) {
          __nv_bfloat16* kcache = reinterpret_cast<__nv_bfloat16*>(P.key_cache) + head_block;
          kcache[(static_cast<size_t>(i0 >> 3) * seq_len + pos) * 8 + (i0 & 7)] = __float2bfloat16_rn(r0);
          kcache[(static_cast<size_t>(i1 >> 3) * seq_len + pos) * 8 + (i1 & 7)] = __float2bfloat16_rn(r1);
        } else {
          float* kcache = P.key_cache + head_block;
          kcache[(static_cast<size_t>(i0 >> 2) * seq_len + pos) * 4 + (i0 & 3)] = r0;
          kcache[(static_cast<size_t>(i1 >> 2) * seq_len + pos) * 4 + (i1 & 3)] = r1;
        }
      }
    }
  }
  return need_v ? in.v : 0.f;
}

// ---- attention: SP CTAs per query head, two phases (mha_kernel.cu:47-110 + rope_kernel.cu) ---------
// The reference gives a head one CTA and so did round 1: 32 of the SMs worked while the rest polled,
// and the time grew with the context.  Every score (one left-to-right FFMA chain per timestep) and
// every output element (one FFMA chain over the timesteps) is independent of the others, so the work
// splits over SP CTAs per head WITHOUT touching a single chain -- results stay bit-identical:
//   scores phase  CTA (head, s) rotates q (and the new key row), takes the K tiles j = s, s + SP, ...
//                 and publishes its scaled scores as tagged words scores[head][t];
//   P.V phase     CTA (head, s) polls all pos + 1 scores of the head, runs the softmax (every CTA of
//                 the head the same bits), and owns output dims [s dv, (s + 1) dv), dv = head_size / SP:
//                 it streams only that slice of V and publishes its dv outputs.
// KV layout (persistent engine only; kllm_decoder_read_kv converts back):
//   K [L][kv_head][head_size/4][seq_len][4]   -- 16-byte chunk c of timestep t at ((c*seq_len)+t)*4:
//       a tile of T timesteps is hs/4 contiguous runs of T*16 bytes, and "thread t reads chunk c"
//       is a conflict-free 128-bit shared-memory access (consecutive t -> consecutive 16 B);
//   V [L][kv_head][SP][seq_len][dv]           -- a tile of T timesteps of one slice is one contiguous
//       block and "thread i walks column i" is conflict-free.
//   bf16 KV cache (flash form, SP layout 1): K [L][kv_head][head_size/8][seq_len][8] and V [L][kv_head][seq_len]
//       [head_size] in bf16 -- still 16-byte chunks and contiguous V rows, half the bytes.
//   fp8 KV cache (the same form): K [L][kv_head][head_size/16][seq_len][16] and V [L][kv_head][seq_len][head_size]
//       in e4m3 codes -- a quarter of the bytes.
// Rows t < pos were written by earlier tokens, so -- like weights -- the producer warp streams
// them through the ring ahead of time; only row pos is handled here from registers.
__device__ __forceinline__ int attn_tiles(int pos, int T) { return (pos + T - 1) / T; }
// tiles j = s, s + SP, ... < n
__device__ __forceinline__ int own_tiles(int n, int s, int SP) { return n > s ? (n - s + SP - 1) / SP : 0; }

// One output element's P.V chain over nt timesteps of a staged tile: value += pr[tt] * vt[tt * stride],
// strictly left to right (mha_kernel.cu:97-109).  The chain is latency bound (one dependent FFMA per
// step), so the operands of the next eight steps are loaded while the current eight retire.
// pv_chain_smem: probabilities in shared memory (the usual case) -- explicit ld.shared, the eight
// probabilities of a batch as two 128-bit loads (pr_addr is 16-byte aligned: tiles start at
// multiples of 32 timesteps).  pv_chain: probabilities behind a generic pointer (global fallback).
__device__ __forceinline__ float pv_chain_smem(uint32_t pr_addr, uint32_t vt_addr, int stride_bytes, int nt, float value) {
  // two register sets (A: steps tt .. tt+7, B: tt+8 .. tt+15) loaded alternately, so the loop carries no
  // register moves and every load has a whole 8-step chain (>= 32 cycles) to land
  auto load8 = [&](int t, float4& p0, float4& p1, float (&v)[8]) {
    p0 = lds_f4(pr_addr + t * 4), p1 = lds_f4(pr_addr + t * 4 + 16);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = lds_f32(vt_addr + (t + k) * stride_bytes);
  };
  auto chain8 = [&](const float4& p0, const float4& p1, const float (&v)[8]) {
    value = __fmaf_rn(p0.x, v[0], value);
    value = __fmaf_rn(p0.y, v[1], value);
    value = __fmaf_rn(p0.z, v[2], value);
    value = __fmaf_rn(p0.w, v[3], value);
    value = __fmaf_rn(p1.x, v[4], value);
    value = __fmaf_rn(p1.y, v[5], value);
    value = __fmaf_rn(p1.z, v[6], value);
    value = __fmaf_rn(p1.w, v[7], value);
  };
  int tt = 0;
  if (nt >= 8) {
    float4 a0, a1, b0, b1;
    float va[8], vb[8];
    load8(0, a0, a1, va);
    for (; tt + 24 <= nt; tt += 16) {  // A holds tt .. tt+7
      load8(tt + 8, b0, b1, vb);
      chain8(a0, a1, va);
      load8(tt + 16, a0, a1, va);
      chain8(b0, b1, vb);
    }
    if (tt + 16 <= nt) {
      load8(tt + 8, b0, b1, vb);
      chain8(a0, a1, va);
      chain8(b0, b1, vb);
      tt += 16;
    } else {
      chain8(a0, a1, va);
      tt += 8;
    }
  }
  for (; tt < nt; ++tt) value = __fmaf_rn(lds_f32(pr_addr + tt * 4), lds_f32(vt_addr + tt * stride_bytes), value);
  return value;
}
__device__ __forceinline__ float pv_chain(const float* pr, const float* vt, int stride, int nt, float value) {
#pragma unroll 8
  for (int tt = 0; tt < nt; ++tt) value = __fmaf_rn(pr[tt], vt[tt * stride], value);
  return value;
}

// ---- exact attention: the pieces the fused and the split forms share ---------------------------------------
// One timestep's score, q . k over head_size as one left-to-right FFMA chain (mha_kernel.cu:61-91): k4[c * stride]
// is the 16-byte chunk c of the timestep -- stride T in a staged K tile, 1 for the freshly rotated key.
__device__ __forceinline__ float qk_chain(const float4* k4, int stride, const float4* q4, int hs) {
  float score = 0.0f;
#pragma unroll 4
  for (int c = 0; c < (hs >> 2); ++c) {
    const float4 kv = k4[c * stride];
    const float4 qv = q4[c];
    score = __fmaf_rn(kv.x, qv.x, score);
    score = __fmaf_rn(kv.y, qv.y, score);
    score = __fmaf_rn(kv.z, qv.z, score);
    score = __fmaf_rn(kv.w, qv.w, score);
  }
  return score;
}

// The scaled scores of the K tiles j = j0, j0 + SP, ... (thread t < nt takes timestep t0 + t of a tile) and, in the
// CTA with j0 == 0, thread 0's score of pos from the freshly rotated key.  store(t, score) puts one away.  With
// `timed`, c_wait gathers the cycles spent waiting for tiles.
template <typename Store>
__device__ __forceinline__ void exact_scores(const Params& P, const float* q_s, const float* k_s, int j0, int SP,
                                             int pos, Pipe& pipe, bool timed, long long& c_wait, Store store) {
  const unsigned char* stages = smem + P.xbuf_bytes + P.xres_bytes;
  const int tid = threadIdx.x;
  const int hs = P.head_size, T = P.attn_tile, S = P.num_stages;
  const float scale = 1.f / sqrtf(static_cast<float>(hs));
  const float4* q4 = reinterpret_cast<const float4*>(q_s);
  const int n_tiles = attn_tiles(pos, T);
  for (int j = j0; j < n_tiles; j += SP) {
    const int t0 = j * T;
    const int nt = min(T, pos - t0);
    const long long w0 = timed ? clock64() : 0;
    mbar_wait(&g_full_bar[pipe.slot], pipe.parity);
    if (timed) c_wait += clock64() - w0;
    const float4* tile = reinterpret_cast<const float4*>(stages + static_cast<size_t>(pipe.slot) * P.stage_bytes);
    if (tid < nt) store(t0 + tid, __fmul_rn(qk_chain(tile + tid, T, q4, hs), scale));
    __syncwarp();
    if ((tid & 31) == 0) mbar_arrive(&g_empty_bar[pipe.slot]);
    pipe.advance(S);
  }
  if (j0 == 0 && tid == 0) store(pos, __fmul_rn(qk_chain(reinterpret_cast<const float4*>(k_s), 1, q4, hs), scale));
}

// The softmax of score_head[0 .. size) in place, mha_kernel.cu:7-45: the reference runs 256 strided threads and
// cub<256> block reductions.  Here 128 threads play two virtual threads each (v = tid and v = tid + 128, i.e.
// elements tid + 256 k and tid + 128 + 256 k): the maximum does not care about order, and for the sum each virtual
// thread keeps its own left-to-right partial, each virtual warp its own shuffle tree (real warp q holds virtual
// warps q and q + 4), then the eight warp sums are added in order.  Every CTA that runs it gets the same bits.
__device__ __forceinline__ void exact_softmax(float* score_head, int size) {
  constexpr int kHalf = kSoftmaxThreads / 2;  // 128 real threads
  static_assert(kConsumerThreads >= kHalf, "softmax needs 128 consumer threads");
  float* s_warp = g_s_warp;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool sm_thread = tid < kHalf;
  float max_val = -FLT_MAX;
  if (sm_thread)
    for (int i = tid; i < size; i += kHalf) max_val = fmaxf(max_val, score_head[i]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) max_val = fmaxf(max_val, __shfl_xor_sync(kFull, max_val, off));
  if (lane == 0 && sm_thread) s_warp[warp] = max_val;
  consumer_sync();
  max_val = fmaxf(fmaxf(s_warp[0], s_warp[1]), fmaxf(s_warp[2], s_warp[3]));
  consumer_sync();

  float sum_lo = 0.0f, sum_hi = 0.0f;  // virtual threads tid and tid + 128
  if (sm_thread) {
    for (int i = tid; i < size; i += kSoftmaxThreads) {
      const float e = expf(score_head[i] - max_val);
      score_head[i] = e;
      sum_lo += e;
    }
    for (int i = tid + kHalf; i < size; i += kSoftmaxThreads) {
      const float e = expf(score_head[i] - max_val);
      score_head[i] = e;
      sum_hi += e;
    }
  }
  sum_lo = warp_tree_sum(sum_lo);
  sum_hi = warp_tree_sum(sum_hi);
  if (lane == 0 && sm_thread) {
    s_warp[warp] = sum_lo;      // virtual warp `warp`
    s_warp[warp + 4] = sum_hi;  // virtual warp `warp + 4`
  }
  consumer_sync();
  if (tid == 0) {
    float total = s_warp[0];
#pragma unroll
    for (int w = 1; w < kSoftmaxThreads / 32; ++w) total = __fadd_rn(total, s_warp[w]);
    g_s_bcast = total;
  }
  consumer_sync();
  const float sum = g_s_bcast;
  for (int i = tid; i < size; i += kConsumerThreads) score_head[i] = score_head[i] / sum;
  consumer_sync();
}

// Output dim tid < dv of P.V, mha_kernel.cu:97-109: one FFMA chain over the V tiles of the CTA's slice ([T][dv]
// each), ending with the current position's probability times v_pos.  score_head holds the probabilities, in
// shared memory when score_in_smem.  With `timed`, c_wait gathers the cycles spent waiting for tiles.
__device__ __forceinline__ float exact_pv(const Params& P, const float* score_head, bool score_in_smem, int dv, int pos,
                                          float v_pos, Pipe& pipe, bool timed, long long& c_wait) {
  const unsigned char* stages = smem + P.xbuf_bytes + P.xres_bytes;
  const int tid = threadIdx.x;
  const int T = P.attn_tile_v, S = P.num_stages;
  float value = 0.0f;
  const int n_tiles = attn_tiles(pos, T);
  for (int j = 0; j < n_tiles; ++j) {
    const int t0 = j * T;
    const int nt = min(T, pos - t0);
    const long long w0 = timed ? clock64() : 0;
    mbar_wait(&g_full_bar[pipe.slot], pipe.parity);
    if (timed) c_wait += clock64() - w0;
    if (tid < dv) {
      const float* vt = reinterpret_cast<const float*>(stages + static_cast<size_t>(pipe.slot) * P.stage_bytes) + tid;
      value = score_in_smem ? pv_chain_smem(smem_u32(score_head + t0), smem_u32(vt), dv * 4, nt, value)
                            : pv_chain(score_head + t0, vt, dv, nt, value);
    }
    __syncwarp();
    if ((tid & 31) == 0) mbar_arrive(&g_empty_bar[pipe.slot]);
    pipe.advance(S);
  }
  if (tid < dv) value = __fmaf_rn(score_head[pos], v_pos, value);
  return value;
}

// Fused form (attn_split == 1, one CTA per head does scores, softmax and P.V in ONE phase): one
// hand-off less per layer, the better trade when a head's K and V are small (head_size 64).
__device__ KLLM_PHASE_CALL Pipe attention_fused_phase(const Params& P, int head, int pos, Pipe pipe, unsigned tag_in,
                                                 unsigned tag_out, unsigned long long* stamp) {
  const Phase& ph = g_ph_cons;
  float* ws = reinterpret_cast<float*>(smem);
  const int tid = threadIdx.x;
  const long long c_begin = stamp ? clock64() : 0;
  long long c_wait = 0;
  const int hs = P.head_size, seq_len = P.seq_len;
  float* q_s = ws;       // [hs] rotated query
  float* k_s = ws + hs;  // [hs] rotated key of the current position
  const int kvh = head / P.kv_mul;
  const size_t head_block = (static_cast<size_t>(ph.layer) * (P.kv_dim / hs) + kvh) * seq_len * hs;
  // scores / probabilities: shared memory when the context fits the workspace (the ring leaves
  // almost no L1), else the global [head][seq_len] buffer the reference uses
  const int smem_cap = (P.xbuf_bytes >> 2) - 2 * hs;
  const bool score_in_smem = pos + 1 <= smem_cap;
  float* score_head = score_in_smem ? (ws + 2 * hs) : (P.score + static_cast<size_t>(head) * seq_len);

  // q, the new key row (rotated) and the value row of the current position (QKV phase of this token)
  const float v_pos = attention_inputs(P, ph, head, kvh, pos, tag_in, true, true, q_s, k_s, head_block);
  consumer_sync();
  const long long c_rope = stamp ? clock64() : 0;
  exact_scores(P, q_s, k_s, 0, 1, pos, pipe, stamp != nullptr, c_wait, [&](int t, float s) { score_head[t] = s; });
  consumer_sync();
  const long long c_scores = stamp ? clock64() : 0;
  const long long c_wait_scores = c_wait;
  exact_softmax(score_head, pos + 1);
  const long long c_soft = stamp ? clock64() : 0;
  const float value = exact_pv(P, score_head, score_in_smem, hs, pos, v_pos, pipe, stamp != nullptr, c_wait);
  if (tid < hs) st_tagged_gpu(ph.ta + static_cast<size_t>(head) * hs + tid, value, tag_out);
  if (stamp && tid == 0) {  // SM cycles of thread 0 (tools/phase_timeline.py)
    const long long c_end = clock64();
    stamp[4] = static_cast<unsigned long long>(c_rope - c_begin);                             // q/k/v poll + RoPE
    stamp[5] = static_cast<unsigned long long>(c_scores - c_rope - c_wait_scores);            // scores
    stamp[6] = static_cast<unsigned long long>(c_soft - c_scores);                            // softmax
    stamp[7] = static_cast<unsigned long long>(c_end - c_soft - (c_wait - c_wait_scores));    // P.V
    stamp[8] = static_cast<unsigned long long>(c_wait);                                       // ring waits
    stamp[9] = static_cast<unsigned long long>(c_wait - c_wait_scores);                       // of which V tiles
  }
  return pipe;
}

__device__ KLLM_PHASE_CALL Pipe attention_scores_phase(const Params& P, int head, int split, int pos, Pipe pipe,
                                                        unsigned tag_in, unsigned tag_out, unsigned long long* stamp) {
  const Phase& ph = g_ph_cons;
  float* ws = reinterpret_cast<float*>(smem);
  const int tid = threadIdx.x;
  const long long c_begin = stamp ? clock64() : 0;
  long long c_wait = 0;
  const int hs = P.head_size, seq_len = P.seq_len;
  float* q_s = ws;       // [hs] rotated query
  float* k_s = ws + hs;  // [hs] rotated key of the current position
  const int kvh = head / P.kv_mul;
  const size_t head_block = (static_cast<size_t>(ph.layer) * (P.kv_dim / hs) + kvh) * seq_len * hs;
  unsigned long long* sc_out = P.scores + static_cast<size_t>(head) * seq_len;
  // q and -- in the CTA that scores it -- the new key row, rotated (the value row is the P.V phase's business)
  attention_inputs(P, ph, head, kvh, pos, tag_in, split == 0, false, q_s, k_s, head_block);
  consumer_sync();
  const long long c_rope = stamp ? clock64() : 0;
  exact_scores(P, q_s, k_s, split, P.attn_split, pos, pipe, stamp != nullptr, c_wait,
               [&](int t, float s) { st_tagged_gpu(sc_out + t, s, tag_out); });
  if (stamp && tid == 0) {
    const long long c_end = clock64();
    stamp[4] = static_cast<unsigned long long>(c_rope - c_begin);           // q/k poll + RoPE
    stamp[5] = static_cast<unsigned long long>(c_end - c_rope - c_wait);    // scores
    stamp[8] = static_cast<unsigned long long>(c_wait);                     // ring waits (K tiles)
  }
  return pipe;
}

__device__ KLLM_PHASE_CALL Pipe attention_pv_phase(const Params& P, int head, int split, int pos, Pipe pipe,
                                                   unsigned tag_scores, unsigned tag_qkv, unsigned tag_out,
                                                   unsigned long long* stamp) {
  const Phase& ph = g_ph_cons;
  float* ws = reinterpret_cast<float*>(smem);
  const int tid = threadIdx.x;
  const long long c_begin = stamp ? clock64() : 0;
  long long c_wait = 0;
  const int hs = P.head_size, seq_len = P.seq_len;
  const int dv = hs / P.attn_split;
  const int kvh = head / P.kv_mul;
  // scores / probabilities: shared memory when the context fits the workspace (the ring leaves
  // almost no L1), else this CTA's own global row: the softmax rewrites its row in place, so a row shared by the
  // SP CTAs of a head would let one CTA read the other's exponentials as scores
  const int smem_cap = P.xbuf_bytes >> 2;
  const bool score_in_smem = pos + 1 <= smem_cap;
  float* score_head =
      score_in_smem ? ws : (P.probs + (static_cast<size_t>(head) * P.attn_split + split) * seq_len);

  // this CTA's dv dims of the value row of the current position (written by the QKV phase of this token)
  float v_pos = 0.f;
  if (tid < dv) v_pos = poll_tagged(ph.tv + kvh * hs + split * dv + tid, tag_qkv);

  // all pos + 1 scaled scores of the head, polled in place
  const int size = pos + 1;
  {
    const unsigned long long* sc_in = P.scores + static_cast<size_t>(head) * seq_len;
    const int n4 = size >> 2;  // seq_len % 4 == 0: the head's words start 32-byte aligned
    stage_handoff<4>(sc_in, tag_scores, n4, tid, kConsumerThreads, reinterpret_cast<float4*>(score_head));
    const int rest = 4 * n4 + tid;
    if (tid < 4 && rest < size) score_head[rest] = poll_tagged(sc_in + rest, tag_scores);
  }
  consumer_sync();
  const long long c_poll = stamp ? clock64() : 0;
  exact_softmax(score_head, size);
  const long long c_soft = stamp ? clock64() : 0;
  const float value = exact_pv(P, score_head, score_in_smem, dv, pos, v_pos, pipe, stamp != nullptr, c_wait);
  if (tid < dv) st_tagged_gpu(ph.ta + static_cast<size_t>(head) * hs + split * dv + tid, value, tag_out);
  if (stamp && tid == 0) {
    const long long c_end = clock64();
    stamp[4] = static_cast<unsigned long long>(c_poll - c_begin);           // scores (+ v row) polled
    stamp[6] = static_cast<unsigned long long>(c_soft - c_poll);            // softmax
    stamp[7] = static_cast<unsigned long long>(c_end - c_soft - c_wait);    // P.V
    stamp[8] = static_cast<unsigned long long>(c_wait);                     // ring waits (V tiles)
  }
  return pipe;
}

// Toleranced attention (numerics "fast"): flash-decoding.  With the summation order free, a head is
// split over SP CTAs BY TIMESTEP -- CTA (head, s) takes the tiles j = s, s + SP, ... of T timesteps, K
// and V -- and inside the CTA every WARP runs its own online softmax over blocks of 8 timesteps
// (blocks dealt round-robin to the warps), so a tile costs no block-wide barrier at all:
//   scores   lane (cg, tt) = (lane / 8, lane % 8) dots timestep tt of the block with a quarter of
//            head_size (conflict-free 128-bit reads of the K tile [hs/4][T][4]); two xor-shuffles sum
//            the quarters, three more give the block's maximum and sum -> running (m, l) of the warp;
//   P.V      lane owns output dims lane, lane + 32, ...: o[d] = o[d] alpha + sum_tt p_tt v[tt][d] with p_tt
//            shuffled from lane tt (conflict-free 32-bit reads of the V tile [T][hs]).
// bf16 KV cache (KV16): the same mapping over tiles of half the bytes -- a 16-byte K chunk is 8 dims of a
// timestep (K tile [hs/8][T][8], so a quarter of the head is hs/32 chunks) and the V tile is [T][hs] bf16;
// every element is widened exactly to fp32 and the arithmetic is unchanged.
// fp8 KV cache: a 16-byte K chunk is 16 dims (a quarter of the head is hs/64 chunks, host: head_size % 64 == 0) and
// the V tile is [T][hs] e4m3 codes; each code widens exactly to value(code), the K scale s_k is folded into the
// cached rows' score scale and the V scale s_v into the warp partials o[] (the row of pos, from registers, is
// unscaled).
// At the end the warp partials (m, l, o[hs]) are merged through shared memory, CTA 0 of the head folds
// in the current position's row from registers and merges the partials of the other CTAs that had
// tiles (tagged words in the scores area: [head][s][hs + 2]); at short contexts (pos <= T) that is
// nobody, and the phase costs what the fused one does.
template <int KV>
__device__ KLLM_PHASE_CALL Pipe attention_flash_phase(const Params& P, int head, int split, int pos, Pipe pipe,
                                                       unsigned tag_in, unsigned tag_out, unsigned long long* stamp) {
  const Phase& ph = g_ph_cons;
  float* ws = reinterpret_cast<float*>(smem);
  unsigned char* stages = smem + P.xbuf_bytes + P.xres_bytes;
  uint64_t* full_bar = g_full_bar;
  uint64_t* empty_bar = g_empty_bar;
  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  const long long c_begin = stamp ? clock64() : 0;
  long long c_wait = 0, c_sc = 0, c_pv = 0;
  const int hs = P.head_size, seq_len = P.seq_len, T = P.attn_tile, S = P.num_stages, SP = P.attn_split;
  const int n_tiles = attn_tiles(pos, T);
  // CTAs without a tile have nothing to say (their partial would weigh zero): only CTA 0 always runs
  if (split != 0 && split >= n_tiles) return pipe;
  float* q_s = ws;                // [hs] rotated query
  float* k_s = ws + hs;           // [hs] rotated key of the current position
  float* red = ws + 2 * hs;       // [kConsumerWarps][hs + 2] warp partials: m, l, o[hs]
  const int kvh = head / P.kv_mul;
  const size_t head_block = (static_cast<size_t>(ph.layer) * (P.kv_dim / hs) + kvh) * seq_len * hs;
  // q, and in CTA 0 of the head the new key row (rotated) and the value row of the current position
  const float v_pos = attention_inputs<KV>(P, ph, head, kvh, pos, tag_in, split == 0, split == 0, q_s, k_s, head_block);
  consumer_sync();
  const long long c_rope = stamp ? clock64() : 0;

  constexpr bool KV16 = KV == KLLM_KV_BF16, KV8 = KV == KLLM_KV_FP8;
  const float scale = 1.f / sqrtf(static_cast<float>(hs));
  // the cached rows' score scale: with the fp8 cache s_k folded in
  float tile_scale = scale;
  if constexpr (KV8) tile_scale = scale * P.kv_scale_k[ph.layer * (P.kv_dim / hs) + kvh];
  const float4* q4 = reinterpret_cast<const float4*>(q_s);
  const int cg = lane >> 3, tt = lane & 7;
  const int cpg = hs >> 4;        // 16-byte chunks per quarter of head_size (host: head_size % 16 == 0)
  float m = -FLT_MAX, l = 0.f;
  float o[4] = {0.f, 0.f, 0.f, 0.f};  // output dims lane, lane + 32, lane + 64, lane + 96 (< hs)
  int blk0 = 0;                   // blocks dealt so far: block b of the CTA goes to warp b % kConsumerWarps
  for (int j = split; j < n_tiles; j += SP) {
    const int t0 = j * T;
    const int nt = min(T, pos - t0);
    const long long w0 = stamp ? clock64() : 0;
    mbar_wait(&full_bar[pipe.slot], pipe.parity);  // K tile
    const uint32_t ktile = smem_u32(stages + static_cast<size_t>(pipe.slot) * P.stage_bytes);
    const int kslot = pipe.slot;
    pipe.advance(S);
    mbar_wait(&full_bar[pipe.slot], pipe.parity);  // V tile
    const uint32_t vtile = smem_u32(stages + static_cast<size_t>(pipe.slot) * P.stage_bytes);
    const long long w1 = stamp ? clock64() : 0;
    c_wait += w1 - w0;
    const int nb = (nt + 7) >> 3;
    for (int b = (warp - blk0 % kConsumerWarps + kConsumerWarps) % kConsumerWarps; b < nb;
         b += kConsumerWarps) {
      const long long s0 = stamp ? clock64() : 0;
      const int tl = b * 8 + tt;  // this lane's timestep within the tile
      const bool valid = tl < nt;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      if (KV8 && valid) {  // chunk c = dims 16c .. 16c + 15 of the timestep, 16 e4m3 codes (host: head_size % 64 == 0)
#pragma unroll 2
        for (int c = cg * (cpg >> 2); c < (cg + 1) * (cpg >> 2); ++c) {
          const float4 kw = lds_f4(ktile + static_cast<uint32_t>(c * T + tl) * 16u);
          const float kword[4] = {kw.x, kw.y, kw.z, kw.w};
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            const float4 kv = e4m3x4_values(__float_as_uint(kword[w]));
            const float4 qv = q4[4 * c + w];
            a0 = __fmaf_rn(kv.x, qv.x, a0);
            a1 = __fmaf_rn(kv.y, qv.y, a1);
            a2 = __fmaf_rn(kv.z, qv.z, a2);
            a3 = __fmaf_rn(kv.w, qv.w, a3);
          }
        }
      } else if (KV16 && valid) {  // chunk c = dims 8c .. 8c + 7 of the timestep, 8 bf16 (host: head_size % 32 == 0)
#pragma unroll 2
        for (int c = cg * (cpg >> 1); c < (cg + 1) * (cpg >> 1); ++c) {
          const float4 kw = lds_f4(ktile + static_cast<uint32_t>(c * T + tl) * 16u);
          const float4 qa = q4[2 * c], qb = q4[2 * c + 1];
          a0 = __fmaf_rn(bf16_lo(kw.x), qa.x, a0);
          a1 = __fmaf_rn(bf16_hi(kw.x), qa.y, a1);
          a2 = __fmaf_rn(bf16_lo(kw.y), qa.z, a2);
          a3 = __fmaf_rn(bf16_hi(kw.y), qa.w, a3);
          a0 = __fmaf_rn(bf16_lo(kw.z), qb.x, a0);
          a1 = __fmaf_rn(bf16_hi(kw.z), qb.y, a1);
          a2 = __fmaf_rn(bf16_lo(kw.w), qb.z, a2);
          a3 = __fmaf_rn(bf16_hi(kw.w), qb.w, a3);
        }
      } else if (valid) {
#pragma unroll 4
        for (int c = cg * cpg; c < (cg + 1) * cpg; ++c) {
          const float4 kv = lds_f4(ktile + static_cast<uint32_t>(c * T + tl) * 16u);
          const float4 qv = q4[c];
          a0 = __fmaf_rn(kv.x, qv.x, a0);
          a1 = __fmaf_rn(kv.y, qv.y, a1);
          a2 = __fmaf_rn(kv.z, qv.z, a2);
          a3 = __fmaf_rn(kv.w, qv.w, a3);
        }
      }
      float sc = (a0 + a1) + (a2 + a3);
      sc += __shfl_xor_sync(kFull, sc, 8);
      sc += __shfl_xor_sync(kFull, sc, 16);
      sc = valid ? sc * tile_scale : -FLT_MAX;
      float mb = sc;
      mb = fmaxf(mb, __shfl_xor_sync(kFull, mb, 1));
      mb = fmaxf(mb, __shfl_xor_sync(kFull, mb, 2));
      mb = fmaxf(mb, __shfl_xor_sync(kFull, mb, 4));
      const float m_new = fmaxf(m, mb);
      const float alpha = expf(m - m_new);
      const float pr = valid ? expf(sc - m_new) : 0.f;
      float ps = pr;
      ps += __shfl_xor_sync(kFull, ps, 1);
      ps += __shfl_xor_sync(kFull, ps, 2);
      ps += __shfl_xor_sync(kFull, ps, 4);
      l = __fmaf_rn(l, alpha, ps);
      m = m_new;
      const long long s1 = stamp ? clock64() : 0;
      c_sc += s1 - s0;
      // P.V of the block
      const int nv = min(8, nt - b * 8);
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      // element (timestep, dim) of the V tile [T][hs] at byte (timestep * hs + dim) << esh: the 32 lanes read
      // 32 consecutive elements, conflict-free in either width
      constexpr uint32_t esh = KV8 ? 0u : KV16 ? 1u : 2u;
      const uint32_t vrow = vtile + (static_cast<uint32_t>(b * 8 * hs + lane) << esh);
      for (int k = 0; k < nv; ++k) {
        const float pk = __shfl_sync(kFull, pr, k);
        const uint32_t va = vrow + (static_cast<uint32_t>(k * hs) << esh);
#pragma unroll
        for (int i = 0; i < 4; ++i)
          if (lane + 32 * i < hs) {
            const uint32_t a = va + ((32u * i) << esh);
            acc[i] = __fmaf_rn(pk, KV8 ? lds_e4m3(a) : KV16 ? lds_bf16(a) : lds_f32(a), acc[i]);
          }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = __fmaf_rn(o[i], alpha, acc[i]);
      if (stamp) c_pv += clock64() - s1;
    }
    blk0 += nb;
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&empty_bar[kslot]);
      mbar_arrive(&empty_bar[pipe.slot]);
    }
    pipe.advance(S);
  }
  const long long c_tiles = stamp ? clock64() : 0;
  // ---- merge the warps' partials: thread d < hs ends with the CTA's (m, l, o[d]) ---------------------
  {
    float* mine = red + warp * (hs + 2);
    if (lane == 0) mine[0] = m, mine[1] = l;
    if constexpr (KV8) {  // the cached rows' values times s_v
      const float sv = P.kv_scale_v[ph.layer * (P.kv_dim / hs) + kvh];
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = __fmul_rn(o[i], sv);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (lane + 32 * i < hs) mine[2 + lane + 32 * i] = o[i];
  }
  consumer_sync();
  if (tid < hs) {
    float M = red[0];
    for (int w = 1; w < kConsumerWarps; ++w) M = fmaxf(M, red[w * (hs + 2)]);
    float num = 0.f, den = 0.f;
    for (int w = 0; w < kConsumerWarps; ++w) {
      const float* theirs = red + w * (hs + 2);
      const float wgt = expf(theirs[0] - M);
      num = __fmaf_rn(theirs[2 + tid], wgt, num);
      den = __fmaf_rn(theirs[1], wgt, den);
    }
    if (split == 0) {  // the current position, from the freshly rotated key and the polled value row
      const float4* k4 = reinterpret_cast<const float4*>(k_s);
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      for (int c = 0; c < (hs >> 2); ++c) {
        const float4 kv = k4[c];
        const float4 qv = q4[c];
        a0 = __fmaf_rn(kv.x, qv.x, a0);
        a1 = __fmaf_rn(kv.y, qv.y, a1);
        a2 = __fmaf_rn(kv.z, qv.z, a2);
        a3 = __fmaf_rn(kv.w, qv.w, a3);
      }
      const float s_pos = ((a0 + a1) + (a2 + a3)) * scale;
      const float M_new = fmaxf(M, s_pos);
      const float alpha = expf(M - M_new);
      const float pp = expf(s_pos - M_new);
      num = __fmaf_rn(num, alpha, pp * v_pos);
      den = __fmaf_rn(den, alpha, pp);
      M = M_new;
    }
    unsigned long long* area = P.scores + static_cast<size_t>(head) * seq_len;  // [SP][hs + 2] tagged words
    if (split != 0) {
      unsigned long long* mine = area + static_cast<size_t>(split) * (hs + 2);
      st_tagged_gpu(mine + 2 + tid, num, tag_out);
      if (tid == 0) st_tagged2_gpu(mine, M, den, tag_out);
    } else {
      const int active = min(SP, n_tiles);  // CTAs 1 .. active - 1 of the head had tiles
      // their partials, up to three CTAs' (m, l, o[tid]) in flight together: polled one CTA after the other
      // every partial would be another L2 round trip on the layer's critical path
      for (int s0 = 1; s0 < active; s0 += 3) {
        unsigned long long w_m[3], w_l[3], w_o[3];
        const int ns = min(3, active - s0);
        const long long t_start = clock64();
        for (;;) {
          bool ok = true;
          unsigned seen = tag_out;
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const unsigned long long* theirs = area + static_cast<size_t>(s0 + min(k, ns - 1)) * (hs + 2);
            ld_tagged2_gpu(theirs, w_m[k], w_l[k]);
            w_o[k] = ld_tagged_gpu(theirs + 2 + tid);
          }
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            if (tag_of(w_m[k]) != tag_out) ok = false, seen = tag_of(w_m[k]);
            if (tag_of(w_l[k]) != tag_out) ok = false, seen = tag_of(w_l[k]);
            if (tag_of(w_o[k]) != tag_out) ok = false, seen = tag_of(w_o[k]);
          }
          if (ok) break;
          poll_failed(seen, tag_out, t_start, 0);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (k < ns) {  // in CTA order, as before
            const float ms = val_of(w_m[k]), ls = val_of(w_l[k]), os = val_of(w_o[k]);
            const float M_new = fmaxf(M, ms);
            const float fa = expf(M - M_new), fb = expf(ms - M_new);
            num = __fmaf_rn(num, fa, os * fb);
            den = __fmaf_rn(den, fa, ls * fb);
            M = M_new;
          }
        }
      }
      st_tagged_gpu(ph.ta + static_cast<size_t>(head) * hs + tid, num / den, tag_out);
    }
  }
  if (stamp && tid == 0) {
    const long long c_end = clock64();
    stamp[4] = static_cast<unsigned long long>(c_rope - c_begin);  // q/k/v poll + RoPE
    stamp[5] = static_cast<unsigned long long>(c_sc);              // scores + online softmax (warp 0's blocks)
    stamp[6] = static_cast<unsigned long long>(c_end - c_tiles);   // merges: warps, current row, other CTAs
    stamp[7] = static_cast<unsigned long long>(c_pv);              // P.V (warp 0's blocks)
    stamp[8] = static_cast<unsigned long long>(c_wait);            // ring waits
  }
  return pipe;
}

// ---- log-probabilities: this CTA's part (DESIGN.md 5.8) ---------------------------------------------
// L1 of sampling.cuh over the rows [u0, u1) this CTA produced (or gathered) -- (m_c, S_c) to lp_part[cta] -- and,
// for lp_top_n > 0, their top-N to lp_cand_v / lp_cand_i[cta] (index -1 pads a part of fewer rows).  The input
// vector buffer is idle once every warp is done with its rows (the draw after the barrier relies on the same), so
// it is the scratch.  CTA 0 reads the results behind the token's grid barrier (logprob_record, from
// draw_truncated).
__device__ __noinline__ void logprob_partial(const Params& P, const float* logits, int u0, int u1) {
  auto sync = [] { consumer_sync(); };
  sync();  // the rows of every warp are stored, and no warp reads the input vector any more
  sampling::LogprobScratch& ls = *reinterpret_cast<sampling::LogprobScratch*>(smem);
  const float2 p = sampling::block_part<kConsumerThreads>([&](int i) { return __ldcg(logits + i); }, u0, u1, ls, sync);
  if (threadIdx.x == 0) P.lp_part[blockIdx.x] = p;
  const int N = P.lp_top_n;
  if (N > 0) {
    const size_t off = static_cast<size_t>(blockIdx.x) * sampling::kMaxTopLogprobs;
    sampling::top_n_block<kConsumerThreads>([&](int k) { return sampling::Cand{__ldcg(logits + u0 + k), u0 + k}; },
                                            u1 - u0, N, smem + sampling::kLogprobScratchBase,
                                            P.xbuf_bytes - sampling::kLogprobScratchBase, P.lp_cand_v + off,
                                            P.lp_cand_i + off, sync);
  }
}

// ---- log-probabilities: the record entry (CTA 0, behind the token's grid barrier) --------------------
// L2 over the G parts in CTA order, the top-N of the G x N candidates, then the entry of position `pos` for `id`.
// The input vector buffer is the scratch, as in draw_truncated; the closing barrier orders every read of it before
// the next token stages its first vector.
__device__ __noinline__ void logprob_record(const Params& P, int pos, int id) {
  auto sync = [] { consumer_sync(); };
  sampling::LogprobScratch& ls = *reinterpret_cast<sampling::LogprobScratch*>(smem);
  const int G = gridDim.x, N = P.lp_top_n;
  sync();  // the draw's scratch (the same buffer) is read
  if (threadIdx.x < 32) {
    const float2 f = sampling::warp_fold_parts([&](int c) { return __ldcg(P.lp_part + c); }, G);
    if (threadIdx.x == 0) {
      ls.m = f.x;
      ls.lse_off = f.y;
    }
  }
  if (N > 0) {
    sampling::top_n_block<kConsumerThreads>(
        [&](int k) {
          return sampling::Cand{__ldcg(P.lp_cand_v + (k / N) * sampling::kMaxTopLogprobs + k % N),
                                __ldcg(P.lp_cand_i + (k / N) * sampling::kMaxTopLogprobs + k % N)};
        },
        G * N, N, smem + sampling::kLogprobScratchBase, P.xbuf_bytes - sampling::kLogprobScratchBase, ls.top_v,
        ls.top_i, sync);
  } else {
    sync();
  }
  const size_t row = static_cast<size_t>(pos) * sampling::kMaxTopLogprobs;
  sampling::write_entry(P.logits, P.vocab_size, id, N, ls, P.lp_rec.id + pos, P.lp_rec.lp + pos,
                        P.lp_rec.top_ids + row, P.lp_rec.top_lp + row);
  sync();
}

// ---- the CTA's partial of the draw over its classifier rows -----------------------------------------------
// Over the raw rows [u0, u1) this CTA produced or gathered (stored by its own threads): with LP and the
// log-probabilities on, their partials first (logprob_partial); with step 0 (bias and penalties) on, step 0 of the
// rule, whose adjusted rows go to P.penalized; then the CTA's partial -- greedy, or perturbed as in the
// perturb_only path -- folded over the adjusted rows or else the raw ones.  The rows' mark words in
// P.penalty.marks are this CTA's alone.  draw_truncated reads P.penalized, and the partials stay a lower bound of
// its top-k threshold because they are maxima of the penalised vector.  Each consumer thread t reads only the
// history entries j = t (mod kConsumerThreads), the ones it wrote itself in this launch (the token loop) or that an
// earlier launch wrote, so no hand-off is needed (DESIGN.md 5.7).
template <bool LP>
__device__ __noinline__ ArgBest classifier_partial(const Params& P, const float* logits, int u0, int u1, int pos) {
  if constexpr (LP) {
    if (P.lp_top_n >= 0) logprob_partial(P, logits, u0, u1);
  }
  const SampleParams sp = *P.sampling;
  consumer_sync();  // the raw rows of every warp of the CTA are stored
  const bool step0 = sampling::step0_active(P.penalty);
  if (step0)
    sampling::step0_history<kConsumerThreads>(logits, P.penalized, u0, u1, P.penalty, P.hist, pos,
                                              [] { consumer_sync(); });
  const float* rows = step0 ? P.penalized : logits;
  const bool perturb = sampling::perturb_only(sp, P.vocab_size);
  const uint2 key = sampling::seed_key(sp.seed);
  ArgBest b{0.f, -1};
  for (int i = u0 + static_cast<int>(threadIdx.x); i < u1; i += kConsumerThreads) {
    const float v = __ldcg(rows + i);
    arg_fold(b, perturb ? sampling::perturbed(v, sp.temperature, key, pos, i) : v, i);
  }
  return b;
}

// This CTA's partial of the draw, b of every consumer thread reduced over the warps: to arg_val / arg_idx[cta]
__device__ __forceinline__ void store_cta_partial(const Params& P, ArgBest b) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const float ov = __shfl_xor_sync(kFull, b.v, off);
    const int oi = __shfl_xor_sync(kFull, b.i, off);
    arg_fold(b, ov, oi);
  }
  if (lane == 0) {
    g_s_argv[warp] = b.v;
    g_s_argi[warp] = b.i;
  }
  consumer_sync();
  if (tid == 0) {
    ArgBest c{0.f, -1};
    for (int w = 0; w < kConsumerWarps; ++w) arg_fold(c, g_s_argv[w], g_s_argi[w]);
    P.arg_val[blockIdx.x] = c.v;
    P.arg_idx[blockIdx.x] = c.i;
  }
}

// The greedy id behind the token's grid barrier: a warp folds the G per-CTA partials (argmax_kernel.cu:49-71
// semantics: maximum value, lowest index; every CTA the same).  Sampling without top-k or top-p folds the same
// way: the partials are then the perturbed maxima.
__device__ __forceinline__ int fold_cta_partials(const Params& P) {
  const int lane = threadIdx.x & 31;
  ArgBest b{0.f, -1};
  for (int c = lane; c < static_cast<int>(gridDim.x); c += 32) arg_fold(b, __ldcg(P.arg_val + c), __ldcg(P.arg_idx + c));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float ov = __shfl_xor_sync(kFull, b.v, off);
    const int oi = __shfl_xor_sync(kFull, b.i, off);
    arg_fold(b, ov, oi);
  }
  return b.i < 0 ? 0 : b.i;
}

// The history entry of position `pos`, fed `token`: stored by consumer thread pos % kConsumerThreads of every CTA, the
// one thread that reads it in classifier_partial (-1: an id outside the vocabulary holds none)
__device__ __forceinline__ void record_fed(const Params& P, int pos, int token) {
  if (static_cast<int>(threadIdx.x) == pos % kConsumerThreads)
    P.hist[pos] = static_cast<unsigned>(token) < static_cast<unsigned>(P.vocab_size) ? token : -1;
}

// ---- one GEMV phase of one CTA's consumer warps --------------------------------------------------
// Stages the phase's input vector (tagged residual exchange / tagged hand-off / embedding row) into
// shared memory, RMS-normalises it when the phase asks for it, consumes this CTA's ring stages
// task by task, runs the epilogues and, for the classifier, leaves the CTA's (max, index).
template <WeightFormat F, int KV, bool LP, bool PROF>
__device__ KLLM_PHASE_CALL Carry gemv_phase(const Params& P, Carry carry, int tok, int pos, const float* emb_row,
                                            unsigned long long* stamp) {
  const Phase& ph = g_ph_cons;
  uint64_t* full_bar = g_full_bar;
  uint64_t* empty_bar = g_empty_bar;
  float* s_warp = g_s_warp;
  float* xs = reinterpret_cast<float*>(smem);                  // phase input vector
  float* xres = reinterpret_cast<float*>(smem + P.xbuf_bytes);  // residual stream
  unsigned char* stages = smem + P.xbuf_bytes + P.xres_bytes;
  float4* xs4w = reinterpret_cast<float4*>(xs);
  float4* xres4 = reinterpret_cast<float4*>(xres);
  const float4* xs4 = reinterpret_cast<const float4*>(xs);
  const int S = P.num_stages;
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const int cta = blockIdx.x;
  const int G = gridDim.x;
  Pipe pipe = carry.pipe;
  ArgBest best{carry.best_v, carry.best_i};
  if (!PROF) stamp = nullptr;
  auto hand_tag = [&](int hand) {
    return P.hand_base + static_cast<unsigned>(tok * P.hands_per_token + hand) + 1u;
  };

  // ---- stage the input vector (and RMS-normalise it) --------------------------------------
  const int M = ph.in_dim;
  const int n4 = M >> 2;
  const bool has_norm = ph.norm_w != nullptr;
  float ssq = 0.f;
  bool ssq_ready = false;
  // The RMSNorm weight of the phase does not depend on anything: fetch this thread's packs from L2
  // BEFORE polling the input, so their latency (~0.4 us) hides behind the poll instead of following it.
  // Vectors too long for kNormPre packs per thread are read after the poll as before.  Slots past the end
  // re-read the last pack so that the buffer is always written (stays in registers).
  constexpr int kNormPre = 2;
  const bool norm_pre = has_norm && n4 <= kNormPre * kConsumerThreads;
  float4 nw_pre[kNormPre];
  if (norm_pre) {
    const float4* nw4 = reinterpret_cast<const float4*>(ph.norm_w);
#pragma unroll
    for (int k = 0; k < kNormPre; ++k) nw_pre[k] = __ldg(nw4 + min(tid + k * kConsumerThreads, n4 - 1));
  } else {
#pragma unroll
    for (int k = 0; k < kNormPre; ++k) nw_pre[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (ph.tp_in) {
    // x = x_old + (p_0 + ... + p_{W-1}); no grid barrier, no all-reduce kernel
    const unsigned tag = P.tp_seq_base + static_cast<unsigned>(tok * P.exch_per_token + ph.exch) + 1u;
    const unsigned long long* area =
        P.tp_data[P.tp_rank] + static_cast<size_t>(tag & 1u) * P.tp_world * P.tp_stride;
    switch (P.tp_world) {
      case 1:
        // The 128 rmsnorm threads poll four packs each and fold the sum of squares into the same pass.
        if (has_norm) {
          if (tid < kNormThreads)
            ssq = stage_exchange<1, 4, true>(area, P.tp_stride, tag, n4, tid, kNormThreads, xs4w, xres4);
          ssq_ready = true;
        } else {
          stage_exchange<1, 4, false>(area, P.tp_stride, tag, n4, tid, kConsumerThreads, xs4w, xres4);
        }
        break;
      case 2: stage_exchange<2, 2, false>(area, P.tp_stride, tag, n4, tid, kConsumerThreads, xs4w, xres4); break;
      case 4: stage_exchange<4, 1, false>(area, P.tp_stride, tag, n4, tid, kConsumerThreads, xs4w, xres4); break;
      default: stage_exchange<8, 1, false>(area, P.tp_stride, tag, n4, tid, kConsumerThreads, xs4w, xres4); break;
    }
  } else if (ph.tag_in != nullptr) {
    stage_handoff<4>(ph.tag_in, hand_tag(ph.hand_in), n4, tid, kConsumerThreads, xs4w);
  } else {
    const float4* xg4 = reinterpret_cast<const float4*>(emb_row);
    for (int i = tid; i < n4; i += kConsumerThreads) xs4w[i] = __ldcg(xg4 + i);
  }
  if (stamp) stamp[10] = global_ns();
  if (has_norm) {
    // rmsnorm_kernel.cu:4-50: 128 threads, thread t sums the squares of packs t, t+128, ... with
    // one FFMA chain, cub<128> block reduction, rsqrt(mean + eps), then (scale * x) * w
    if (!ssq_ready) {
      consumer_sync();
      if (tid < kNormThreads)
        for (int p = tid; p < n4; p += kNormThreads) {
          const float4 v = xs4[p];
          ssq = __fmaf_rn(v.x, v.x, ssq);
          ssq = __fmaf_rn(v.y, v.y, ssq);
          ssq = __fmaf_rn(v.z, v.z, ssq);
          ssq = __fmaf_rn(v.w, v.w, ssq);
        }
    }
    if (tid < kNormThreads) {
      const float ws = warp_tree_sum(ssq);
      if (lane == 0) s_warp[warp] = ws;
    }
    consumer_sync();
    const float total = __fadd_rn(__fadd_rn(__fadd_rn(s_warp[0], s_warp[1]), s_warp[2]), s_warp[3]);
    const float sc = rsqrtf(__fadd_rn(__fdiv_rn(total, static_cast<float>(M)), ph.norm_eps));
    {
      // the norm weight (dim floats, the same for every CTA and token) comes from L2 here, once the
      // scale is known: keeping it in registers across the poll made ptxas spill, and with the ring
      // taking all of shared memory a spill is an L2 round trip too
      const float4* nw4 = reinterpret_cast<const float4*>(ph.norm_w);
      auto scale_pack = [&](int i, const float4& nw) {
        float4 v = xs4w[i];
        v.x = __fmul_rn(__fmul_rn(sc, v.x), nw.x);
        v.y = __fmul_rn(__fmul_rn(sc, v.y), nw.y);
        v.z = __fmul_rn(__fmul_rn(sc, v.z), nw.z);
        v.w = __fmul_rn(__fmul_rn(sc, v.w), nw.w);
        xs4w[i] = v;
      };
      if (norm_pre) {
#pragma unroll
        for (int k = 0; k < kNormPre; ++k)
          if (tid + k * kConsumerThreads < n4) scale_pack(tid + k * kConsumerThreads, nw_pre[k]);
      } else {
        for (int i = tid; i < n4; i += kConsumerThreads) scale_pack(i, __ldg(nw4 + i));
      }
    }
  }
  consumer_sync();
  // int8 fast mode: the staged (and normalised) vector becomes 24-bit fixed point per 64-group
  const bool int8_fast = F == WeightFormat::kInt8 && P.int8_fast != 0 && ph.group_size == 64 && (M & 63) == 0;
  if constexpr (F == WeightFormat::kInt8) {
    if (int8_fast) quantize_input_inplace(xs, M, tid);
  }
  if (stamp) stamp[1] = global_ns();

  const int u0 = static_cast<int>(static_cast<long long>(cta) * ph.units / G);
  const int u1 = static_cast<int>(static_cast<long long>(cta + 1) * ph.units / G);
  const int rpu = ph.swiglu ? 2 : 1;
  const int row_bytes = M * weight_bytes(F);

  // the bias of a row is fetched BEFORE its dot product so its L2 latency hides behind the
  // accumulation (by the lane that will run the row's epilogue)
  auto prefetch_addend = [&](int unit, float& bias_v) {
    bias_v = 0.f;
    if (ph.swiglu) return;
    const RowRef rr = resolve_row(ph, unit, 0);
    if (ph.seg[rr.seg].bias != nullptr) bias_v = __ldg(ph.seg[rr.seg].bias + rr.row);
  };
  // one lane per unit
  auto epilogue = [&](int unit, float d0, float d1, float bias_v) {
    if (ph.swiglu) {
      st_tagged_gpu(ph.seg[0].tag_out + unit, swiglu_ref(d0, d1), hand_tag(ph.hand_out));
      return;
    }
    if (ph.tp_out) {
      const unsigned tag = P.tp_seq_base + static_cast<unsigned>(tok * P.exch_per_token + ph.exch_out) + 1u;
      const size_t off = (static_cast<size_t>(tag & 1u) * P.tp_world + P.tp_rank) * P.tp_stride + unit;
      if (P.tp_world == 1) {
        st_tagged_gpu(P.tp_data[0] + off, d0, tag);
      } else {
        for (int k = 1; k <= P.tp_world; ++k) st_tagged(P.tp_data[(P.tp_rank + k) % P.tp_world] + off, d0, tag);
      }
      return;
    }
    const RowRef rr = resolve_row(ph, unit, 0);
    const Seg& sg = ph.seg[rr.seg];
    float v = d0;
    if (sg.bias != nullptr) v = __fadd_rn(v, bias_v);       // matmul.cpp:74-77: out + bias
    if (sg.tag_out != nullptr) st_tagged_gpu(sg.tag_out + rr.row, v, hand_tag(ph.hand_out));
    if (sg.out == nullptr) {
    } else if (sg.head_major) {  // value cache [kv_head][SP][seq_len][dv], bf16 or fp8 elements with those caches
      const int hs = P.head_size, dv = hs / P.attn_vsplit;
      const int kvh = rr.row / hs, d = rr.row % hs;
      const size_t at = ((static_cast<size_t>(kvh) * P.attn_vsplit + d / dv) * P.seq_len + pos) * dv + d % dv;
      if constexpr (KV == KLLM_KV_FP8)
        reinterpret_cast<uint8_t*>(sg.out)[at] = e4m3_encode(v, P.kv_inv_v[ph.layer * (P.kv_dim / hs) + kvh]);
      else if constexpr (KV == KLLM_KV_BF16)
        reinterpret_cast<__nv_bfloat16*>(sg.out)[at] = __float2bfloat16_rn(v);
      else
        sg.out[at] = v;
    } else {
      sg.out[static_cast<long long>(pos) * sg.pos_stride + rr.row] = v;
    }
    if (ph.argmax) arg_fold(best, v, rr.row);
  };

  long long cyc_wait = 0, cyc_rows = 0;
  long long cyc4[4] = {0, 0, 0, 0};
  if (ph.chunks_per_row == 1) {
    // A stage holds n units; they are handed out as tasks of up to 4 rows (plain: 4 units, SwiGLU:
    // 2 units = w1 + w3 rows of two outputs), task after task round-robin over the consumer warps.
    const int ups = ph.rows_per_stage / rpu;
    // Units per task: 4 rows, or 2 SwiGLU units.  The value reaches the loop through an opaque move: with the
    // constant in sight nvcc specialises the loop and the fp32 kernel needs 152 registers instead of 148.
    int upt;
    asm("mov.u32 %0, %1;" : "=r"(upt) : "r"(ph.swiglu ? 2 : 4));
    int task = 0;                      // tasks of this phase so far (same count in every warp)
    for (int u = u0; u < u1; u += ups) {
      const int n = min(ups, u1 - u);
      const long long c0 = stamp ? clock64() : 0;
      mbar_wait(&full_bar[pipe.slot], pipe.parity);
      const long long c1 = stamp ? clock64() : 0;
      cyc_wait += c1 - c0;
      const unsigned char* sbase = stages + static_cast<size_t>(pipe.slot) * P.stage_bytes;
      for (int i0 = 0; i0 < n; i0 += upt, ++task) {
        if (task % kConsumerWarps != warp) continue;
        const int nu = min(upt, n - i0);
        const long long t_a = stamp ? clock64() : 0;
        float bias_v = 0.f;
        if (lane < nu) prefetch_addend(u + i0 + lane, bias_v);
        const long long t_b = stamp ? clock64() : 0;
        float e0 = 0.f, e1 = 0.f;  // this lane's unit: its dot product(s)
        // shared-window addresses of the stage's rows / scale rows
        const uint32_t rb = static_cast<uint32_t>(row_bytes), srb = static_cast<uint32_t>(ph.scale_row_bytes);
        const uint32_t wa = smem_u32(sbase), sa = smem_u32(sbase) + static_cast<uint32_t>(ph.scale_off);
        const uint32_t xa = smem_u32(xs);
        if (ph.swiglu) {
          // stage order: w1 rows of the n units, then their w3 rows
          if (nu == 2) {
            const Rows4 rp{{wa + i0 * rb, wa + (n + i0) * rb, wa + (i0 + 1) * rb, wa + (n + i0 + 1) * rb}};
            const Rows4 sp{{sa + i0 * srb, sa + (n + i0) * srb, sa + (i0 + 1) * srb, sa + (n + i0 + 1) * srb}};
            const float4 d = dot_rows<4, F>(rp, sp, xa, M, ph.group_size, ph.group_shift, lane, int8_fast);
            e0 = lane == 0 ? d.x : d.z;
            e1 = lane == 0 ? d.y : d.w;
          } else {
            const Rows4 rp{{wa + i0 * rb, wa + (n + i0) * rb, 0u, 0u}};
            const Rows4 sp{{sa + i0 * srb, sa + (n + i0) * srb, 0u, 0u}};
            const float4 d = dot_rows<2, F>(rp, sp, xa, M, ph.group_size, ph.group_shift, lane, int8_fast);
            e0 = d.x, e1 = d.y;
          }
        } else if (nu == 4) {
          const Rows4 rp{{wa + i0 * rb, wa + (i0 + 1) * rb, wa + (i0 + 2) * rb, wa + (i0 + 3) * rb}};
          const Rows4 sp{{sa + i0 * srb, sa + (i0 + 1) * srb, sa + (i0 + 2) * srb, sa + (i0 + 3) * srb}};
          const float4 d = dot_rows<4, F>(rp, sp, xa, M, ph.group_size, ph.group_shift, lane, int8_fast);
          e0 = lane == 0 ? d.x : lane == 1 ? d.y : lane == 2 ? d.z : d.w;
        } else {
          int r0 = 0;
          if (nu >= 2) {
            const Rows4 rp{{wa + i0 * rb, wa + (i0 + 1) * rb, 0u, 0u}};
            const Rows4 sp{{sa + i0 * srb, sa + (i0 + 1) * srb, 0u, 0u}};
            const float4 d = dot_rows<2, F>(rp, sp, xa, M, ph.group_size, ph.group_shift, lane, int8_fast);
            e0 = lane == 0 ? d.x : d.y;
            r0 = 2;
          }
          if (r0 < nu) {  // nu is 1 or 3: one more row
            const Rows4 rp{{wa + (i0 + r0) * rb, 0u, 0u, 0u}};
            const Rows4 sp{{sa + (i0 + r0) * srb, 0u, 0u, 0u}};
            const float4 d = dot_rows<1, F>(rp, sp, xa, M, ph.group_size, ph.group_shift, lane, int8_fast);
            if (lane == r0) e0 = d.x;
          }
        }
        const long long t_c = stamp ? clock64() : 0;
        if (lane < nu) epilogue(u + i0 + lane, e0, e1, bias_v);
        if (stamp) {
          cyc4[0] += t_b - t_a, cyc4[1] += t_c - t_b, cyc4[3] += clock64() - t_c;
        }
      }
      __syncwarp();
      if (stamp) cyc_rows += clock64() - c1;
      if (lane == 0) mbar_arrive(&empty_bar[pipe.slot]);
      pipe.advance(S);
    }
  } else {
    // rows longer than a stage (fp32 and bf16): the owning warp carries its partial sums across
    // consecutive stages; chunk boundaries are multiples of 128 packs so every virtual
    // thread still sees its packs in increasing order.  The host never chunks int8 rows; their kernels compile
    // the fp32 loop here.
    constexpr WeightFormat FC = F == WeightFormat::kInt8 ? WeightFormat::kF32 : F;
    for (int u = u0; u < u1; ++u) {
      const bool mine = (u - u0) % kConsumerWarps == warp;
      float bias_v = 0.f;
      if (mine && lane == 0) prefetch_addend(u, bias_v);
      float acc[1][4] = {{0.f, 0.f, 0.f, 0.f}};
      for (int c = 0; c < ph.chunks_per_row; ++c) {
        const int e0 = c * ph.chunk_elems;
        const int ne = min(ph.chunk_elems, M - e0);
        mbar_wait(&full_bar[pipe.slot], pipe.parity);
        if (mine) {
          const uint32_t w[1] = {smem_u32(stages + static_cast<size_t>(pipe.slot) * P.stage_bytes)};
          accum_packs<1, FC>(w, smem_u32(xs) + static_cast<uint32_t>(e0) * 4u, ne >> 2, lane, acc);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[pipe.slot]);
        pipe.advance(S);
      }
      if (mine) {
        const float d0 = block128_sum_vt_packed(acc[0], lane);
        if (lane == 0) epilogue(u, d0, 0.f, bias_v);
      }
    }
  }

  if (ph.argmax) {
    // per-CTA (max, lowest index) of the classifier rows this CTA produced: greedy, the (up to four) lanes that
    // ran epilogues hold partial bests; otherwise the partial is folded anew from the rows the epilogues of this
    // CTA have just stored
    ArgBest wb = best;
    if (sampling::step0_active(P.penalty) || (LP && P.lp_top_n >= 0) || sampling::perturb_only(*P.sampling, P.vocab_size))
      wb = classifier_partial<LP>(P, ph.seg[0].out, u0, u1, pos);
    store_cta_partial(P, wb);
  }
  if (stamp) {
    stamp[2] = global_ns();
    stamp[4] = static_cast<unsigned long long>(cyc4[0]);
    stamp[5] = static_cast<unsigned long long>(cyc4[1]);
    stamp[6] = static_cast<unsigned long long>(cyc4[2]);
    stamp[7] = static_cast<unsigned long long>(cyc4[3]);
    stamp[8] = static_cast<unsigned long long>(cyc_wait);
    stamp[9] = static_cast<unsigned long long>(cyc_rows);
  }
  return Carry{pipe, best.v, best.i};
}

// ---- tensor parallel, classifier sharded by vocabulary ----------------------------------------------
// Rank r computed logits rows [r V/W, (r+1) V/W) and published them as tagged words into EVERY rank's
// exchange area (the tp_out epilogue, exchange `ph.exch`).  Here the CTAs of this rank split the V
// words of the local area between them: poll, store the logit, keep (max, lowest index).  All ranks
// end with the same full logits vector and the same per-CTA partials, hence the same greedy id --
// the cross-rank argmax needs no further exchange.
template <bool LP>
__device__ __noinline__ void gather_logits_phase(const Params& P, int tok, int pos) {
  const Phase& ph = g_ph_cons;
  const int tid = threadIdx.x;
  const int cta = blockIdx.x, G = gridDim.x;
  const int V = ph.units, rows = ph.in_dim;  // rows per rank
  const unsigned tag = P.tp_seq_base + static_cast<unsigned>(tok * P.exch_per_token + ph.exch) + 1u;
  const unsigned long long* area =
      P.tp_data[P.tp_rank] + static_cast<size_t>(tag & 1u) * P.tp_world * P.tp_stride;
  const int u0 = static_cast<int>(static_cast<long long>(cta) * V / G);
  const int u1 = static_cast<int>(static_cast<long long>(cta + 1) * V / G);
  float* logits = ph.seg[0].out;
  const SampleParams sp = *P.sampling;
  const bool perturb = sampling::perturb_only(sp, V);  // as the classifier partials (gemv_phase)
  // with step 0 or the log-probabilities on, the partial is folded afterwards (classifier_partial)
  const bool penalized = sampling::step0_active(P.penalty) || (LP && P.lp_top_n >= 0);
  const uint2 key = sampling::seed_key(sp.seed);
  ArgBest best{0.f, -1};
  for (int i = u0 + tid; i < u1; i += kConsumerThreads) {
    const int r = i / rows, j = i - r * rows;
    const float v = poll_tagged_sys(area + static_cast<size_t>(r) * P.tp_stride + j, tag);
    logits[i] = v;
    if (!penalized) arg_fold(best, perturb ? sampling::perturbed(v, sp.temperature, key, pos, i) : v, i);
  }
  if (penalized) best = classifier_partial<LP>(P, logits, u0, u1, pos);
  store_cta_partial(P, best);
}

// ---- sampled id with top-k or top-p --------------------------------------------------------------
// tau needs all V logits, which are complete in L2 once the classifier's grid barrier is passed.  Every
// CTA draws the id itself from them (no further barrier or hand-off) and gets the same one.  The per-CTA
// maxima of the raw logits that the classifier (or the gather phase) left in arg_val / arg_idx bound the
// top-k tau from below, so only the few logits near the top become candidates; top-p alone takes the
// maximum from them.  The scratch is the input-vector
// buffer: it is idle from the classifier's last read of its input until the next token stages its first
// vector.  The barrier after the draw orders every thread's read of the result
// before any thread writes that buffer again.  With step 0 on, the draw reads the adjusted vector, which is
// complete behind the same barrier (classifier_partial).
__device__ __noinline__ int draw_truncated(const Params& P, int pos) {
  const float* l = sampling::step0_active(P.penalty) ? P.penalized : P.logits;
  const int id = sampling::draw_block<kConsumerThreads>(l, P.vocab_size, *P.sampling, pos, P.arg_val, P.arg_idx,
                                                        static_cast<int>(gridDim.x), smem, P.xbuf_bytes,
                                                        [] { consumer_sync(); });
  consumer_sync();
  return id;
}

// The id of a token in an LP instantiation, and the position's record entry: the draw (top-k / top-p) or the
// kernel's fold of the per-CTA partials, then CTA 0 writes the entry -- of the target teacher[step + 1] when
// scoring.
__device__ __noinline__ int draw_with_logprobs(const Params& P, int pos, int step) {
  const int id = sampling::needs_draw(*P.sampling, P.vocab_size) ? draw_truncated(P, pos) : fold_cta_partials(P);
  if (P.lp_top_n >= 0 && blockIdx.x == 0) logprob_record(P, pos, P.lp_target ? P.teacher[step + 1] : id);
  return id;
}

// ---- the kernel ---------------------------------------------------------------------------------
// decode_megakernel<F, KV, LP, PROF>:
// F: the weight format (fp32, int8 or bf16 rows through the same ring).
// KV: the KV cache's element, a kllm_decoder_desc::kv_cache value -- the bf16 and fp8 caches are fast numerics' flash
// form only.
// LP: launched while log-probabilities are on.  An instantiation with LP false compiles to the code it has without the
// feature: the off path adds nothing to it, not even a test.
// PROF: the stamps of kllm_decoder_profile; they cost registers in the row loops, so only fp32 and int8 weights over
// the fp32 cache have a profiling instantiation.
template <WeightFormat F, int KV, bool LP, bool PROF>
__device__ __forceinline__ void megakernel_body(const Params& P) {
  uint64_t* full_bar = g_full_bar;
  uint64_t* empty_bar = g_empty_bar;
  Phase& s_phase_cons = g_ph_cons;
  Phase& s_phase_prod = g_ph_prod;

  float* xres = reinterpret_cast<float*>(smem + P.xbuf_bytes);  // residual stream
  unsigned char* stages = smem + P.xbuf_bytes + P.xres_bytes;
  const int S = P.num_stages;
  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int warp = tid >> 5;
  const bool is_producer = warp == kConsumerWarps;
  const int cta = blockIdx.x;
  const int G = gridDim.x;

  if (tid == 0) {
    g_stop = 0;
    g_prod_end = 0u;
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  Pipe pipe{0, 0u};
  constexpr int wbytes = weight_bytes(F);

  // =============================== producer warp ===============================================
  if (is_producer) {
    const uint64_t policy = policy_evict_first();  // weights: streamed once per token
    const uint64_t policy_kv = policy_evict_last();  // KV tiles: re-read every token, keep in L2
    int ppos = P.state->pos;
    // The slot of the next fill, of `bytes`: wait until the consumers have released it (null once the run stopped),
    // arm its full barrier with the byte count, and converge the warp, so that a copy by any lane follows the arming.
    // PROF: the cycles each fill of the profiled token waited for a free slot, and the fills, per phase (stamps 11
    // and 12, tools/phase_timeline.py).  A slot is free once the consumers have read it, so this is the time the
    // ring was full: of copies still in flight, or of stages the consumers had not yet read.
    unsigned long long* pstamp = nullptr;
    auto claim_slot = [&](uint32_t bytes) -> unsigned char* {
      const long long pw0 = PROF ? clock64() : 0;
      if (mbar_wait_or_stop(&empty_bar[pipe.slot], pipe.parity ^ 1u, &g_stop)) return nullptr;
      if constexpr (PROF) {
        if (pstamp && lane == 0) {
          atomicAdd(pstamp + 11, static_cast<unsigned long long>(clock64() - pw0));
          atomicAdd(pstamp + 12, 1ull);
        }
      }
      if (lane == 0) mbar_expect_tx(&full_bar[pipe.slot], bytes);
      __syncwarp();
      return stages + static_cast<size_t>(pipe.slot) * P.stage_bytes;
    };
    for (int tok = 0; tok < P.n_tokens; ++tok, ++ppos) {
      const int n_run = tok < P.skip_cls_tokens ? P.n_phases - P.n_cls_phases : P.n_phases;  // prompt token: no classifier
      for (int pi = 0; pi < n_run; ++pi) {
        if constexpr (PROF)
          pstamp = (P.prof != nullptr && tok == P.prof_token)
                       ? P.prof + (static_cast<size_t>(cta) * P.n_phases + pi) * kProfStamps
                       : nullptr;
        {
          const uint32_t* src = reinterpret_cast<const uint32_t*>(P.phases + pi);
          uint32_t* dst = reinterpret_cast<uint32_t*>(&s_phase_prod);
          __syncwarp();
          for (int i = lane; i < static_cast<int>(sizeof(Phase) / 4); i += 32) dst[i] = __ldg(src + i);
          __syncwarp();
        }
        const Phase& ph = s_phase_prod;
        if (ph.kind == kPhaseGather) continue;  // nothing to stream
        if (ph.kind != kPhaseGemv) {
          const int SP = P.attn_split;
          if (cta >= P.head_num * SP || ppos == 0) continue;
          // rows t < pos of this head: final since the previous token.  Order the async-proxy
          // reads after the grid barrier that closed the previous token.
          // (A run that stopped never passes the barrier of the token after the stop: give up then.)
          int stopped = 0;
          if (tok > 0 && lane == 0) {
            const unsigned need = P.barrier_base + static_cast<unsigned>(tok) * static_cast<unsigned>(G);
            while (static_cast<int>(ld_acquire_u32(P.barrier) - need) < 0) {
              if (g_stop) {
                stopped = 1;
                break;
              }
            }
            asm volatile("fence.proxy.async;" ::: "memory");
          }
          if (__shfl_sync(kFull, stopped, 0)) goto producer_done;
          const int hs = P.head_size;
          const int head = cta / SP, split = cta % SP;
          const int kvh = head / P.kv_mul;
          const size_t head_block =
              (static_cast<size_t>(ph.layer) * (P.kv_dim / hs) + kvh) * P.seq_len * hs;
          if (ph.kind == kPhaseAttnFlash) {  // tiles j = split, split + SP, ...: K tile, then V tile
            // K: hs * esz / 16 chunk columns of 16 bytes (4 fp32, 8 bf16 or 16 fp8 dims) per timestep; V: rows of
            // hs * esz
            constexpr int esz = KV == KLLM_KV_FP8 ? 1 : KV == KLLM_KV_BF16 ? 2 : 4;
            const int T = P.attn_tile, row_bytes = hs * esz;
            const unsigned char* kbase = reinterpret_cast<const unsigned char*>(P.key_cache) + head_block * esz;
            const unsigned char* vbase = reinterpret_cast<const unsigned char*>(P.value_cache) + head_block * esz;
            const int n_tiles = attn_tiles(ppos, T);
            for (int j = split; j < n_tiles; j += SP) {
              const int t0 = j * T;
              const int nt = min(T, ppos - t0);
              for (int kv = 0; kv < 2; ++kv) {
                unsigned char* dst = claim_slot(static_cast<uint32_t>(nt) * row_bytes);
                if (dst == nullptr) goto producer_done;
                if (kv == 0) {
                  if (lane < (row_bytes >> 4))
                    bulk_g2s(dst + static_cast<size_t>(lane) * T * 16,
                             kbase + (static_cast<size_t>(lane) * P.seq_len + t0) * 16,
                             static_cast<uint32_t>(nt) * 16, &full_bar[pipe.slot], policy_kv);
                } else if (lane == 0) {
                  bulk_g2s(dst, vbase + static_cast<size_t>(t0) * row_bytes, static_cast<uint32_t>(nt) * row_bytes,
                           &full_bar[pipe.slot], policy_kv);
                }
                pipe.advance(S);
              }
            }
            continue;
          }
          if (ph.kind != kPhaseAttnPV) {  // K tiles j = split, split + SP, ... (fused: SP == 1, all of them)
            const int T = P.attn_tile;
            const float* kbase = P.key_cache + head_block;
            const int n_tiles = attn_tiles(ppos, T);
            for (int j = split; j < n_tiles; j += SP) {
              const int t0 = j * T;
              const int nt = min(T, ppos - t0);
              unsigned char* dst = claim_slot(static_cast<uint32_t>(nt) * hs * 4);
              if (dst == nullptr) goto producer_done;
              if (lane < (hs >> 2))  // hs <= 128 (checked on the host): one 16-byte chunk column per lane
                bulk_g2s(dst + static_cast<size_t>(lane) * T * 16,
                         kbase + (static_cast<size_t>(lane) * P.seq_len + t0) * 4,
                         static_cast<uint32_t>(nt) * 16, &full_bar[pipe.slot], policy_kv);
              pipe.advance(S);
            }
          }
          if (ph.kind != kPhaseAttention) {  // this CTA's slice of V: [seq_len][dv] contiguous
            const int dv = hs / SP, T = P.attn_tile_v;
            const float* vbase = P.value_cache + head_block + static_cast<size_t>(split) * P.seq_len * dv;
            const int n_tiles = attn_tiles(ppos, T);
            for (int j = 0; j < n_tiles; ++j) {
              const int t0 = j * T;
              const int nt = min(T, ppos - t0);
              unsigned char* dst = claim_slot(static_cast<uint32_t>(nt) * dv * 4);
              if (dst == nullptr) goto producer_done;
              if (lane == 0)
                bulk_g2s(dst, vbase + static_cast<size_t>(t0) * dv, static_cast<uint32_t>(nt) * dv * 4,
                         &full_bar[pipe.slot], policy_kv);
              pipe.advance(S);
            }
          }
          continue;
        }
        const int u0 = static_cast<int>(static_cast<long long>(cta) * ph.units / G);
        const int u1 = static_cast<int>(static_cast<long long>(cta + 1) * ph.units / G);
        const int rpu = ph.swiglu ? 2 : 1;
        const int row_bytes = ph.in_dim * wbytes;
        if (ph.chunks_per_row == 1) {
          const int ups = ph.rows_per_stage / rpu;
          for (int u = u0; u < u1; u += ups) {
            const int n = min(ups, u1 - u);
            const int nrows = n * rpu;
            unsigned char* dst = claim_slot(static_cast<uint32_t>(nrows) * (row_bytes + ph.scale_row_bytes));
            if (dst == nullptr) goto producer_done;
            // one bulk copy per run of consecutive rows of one matrix (nrows <= 32: lane = row)
            const RowRef rr = lane < nrows ? stage_row(ph, u, n, lane) : RowRef{-1, -1};
            const int len = run_length(rr, lane, nrows);
            if (len > 0) {
              const long long e = static_cast<long long>(rr.row) * ph.in_dim;
              const unsigned char* src = static_cast<const unsigned char*>(ph.seg[rr.seg].w) + e * wbytes;
              bulk_g2s(dst + static_cast<size_t>(lane) * row_bytes, src, static_cast<uint32_t>(len) * row_bytes,
                       &full_bar[pipe.slot], policy);
              if (ph.scale_row_bytes) {
                const long long g0 = ph.group_shift >= 0 ? (e >> ph.group_shift) : (e / ph.group_size);
                bulk_g2s(dst + ph.scale_off + static_cast<size_t>(lane) * ph.scale_row_bytes,
                         ph.seg[rr.seg].scales + g0, static_cast<uint32_t>(len) * ph.scale_row_bytes,
                         &full_bar[pipe.slot], policy);
              }
            }
            pipe.advance(S);
          }
        } else {
          for (int u = u0; u < u1; ++u) {
            const RowRef rr = resolve_row(ph, u, 0);
            const unsigned char* src = static_cast<const unsigned char*>(ph.seg[rr.seg].w) +
                                       static_cast<long long>(rr.row) * row_bytes;
            for (int c = 0; c < ph.chunks_per_row; ++c) {
              const int e0 = c * ph.chunk_elems;
              const int ne = min(ph.chunk_elems, ph.in_dim - e0);
              unsigned char* dst = claim_slot(static_cast<uint32_t>(ne) * wbytes);
              if (dst == nullptr) goto producer_done;
              if (lane == 0)
                bulk_g2s(dst, src + static_cast<size_t>(e0) * wbytes, static_cast<uint32_t>(ne) * wbytes,
                         &full_bar[pipe.slot], policy);
              pipe.advance(S);
            }
          }
        }
      }
    }
  producer_done:
    // every fill up to here is issued: the consumers of a stopped run drain them before the CTA exits
    if (lane == 0) g_prod_end = 1u + ((static_cast<unsigned>(pipe.slot) << 1) | pipe.parity);
    return;
  }

  // =============================== consumer warps ===============================================
  unsigned bar_target = P.barrier_base;
  int token = P.state->token;
  int pos = P.state->pos;
  record_fed(P, pos, token);
  if (static_cast<unsigned>(token) >= static_cast<unsigned>(P.vocab_size)) token = 0;
  int step = P.state->step;
  float4* xres4 = reinterpret_cast<float4*>(xres);
  constexpr int kPhaseWords = static_cast<int>(sizeof(Phase) / 4);
  static_assert(kPhaseWords <= kConsumerThreads, "phase copy: one word per consumer thread");
  uint32_t next_phase_word = tid < kPhaseWords ? __ldg(reinterpret_cast<const uint32_t*>(P.phases) + tid) : 0u;

  for (int tok = 0; tok < P.n_tokens; ++tok) {
    const float* emb_row = P.tok_emb + static_cast<size_t>(token) * P.dim;
    ArgBest best{0.f, -1};
    // the residual stream starts as the embedding row (llama3.cpp:578-598); the previous token's
    // last reader of xres (classifier staging) is behind the grid barrier that closed that token
    const float4* e4 = reinterpret_cast<const float4*>(emb_row);
    for (int i = tid; i < (P.dim >> 2); i += kConsumerThreads) xres4[i] = __ldg(e4 + i);

    const bool prof_on = PROF && P.prof != nullptr && tok == P.prof_token && tid == 0;
    auto hand_tag = [&](int hand) {
      return P.hand_base + static_cast<unsigned>(tok * P.hands_per_token + hand) + 1u;
    };
    unsigned long long* stamp = nullptr;
    for (int pi = 0; pi < P.n_phases; ++pi) {
      {
        // Fence the CTA's warps before the copy overwrites the descriptor they worked from.  The token's
        // first phase is fenced by the previous token's grid barrier (the first token's by __syncthreads).
        if (pi > 0) consumer_sync();
        uint32_t* dst = reinterpret_cast<uint32_t*>(&s_phase_cons);
        if (tid < kPhaseWords) dst[tid] = next_phase_word;
        consumer_sync();
        // ... and the descriptor of the phase after this one starts its way from L2 now (one word per
        // thread), so that its latency hides behind this phase instead of opening the next
        const int npi = pi + 1 == P.n_phases ? 0 : pi + 1;
        if (tid < kPhaseWords) next_phase_word = __ldg(reinterpret_cast<const uint32_t*>(P.phases + npi) + tid);
      }
      const Phase& ph = s_phase_cons;
      stamp = (PROF && prof_on) ? P.prof + (static_cast<size_t>(cta) * P.n_phases + pi) * kProfStamps : nullptr;
      if (stamp) stamp[0] = global_ns();

      if (ph.kind == kPhaseGather) {
        if (!(tok < P.skip_cls_tokens)) gather_logits_phase<LP>(P, tok, pos);
        if (stamp) stamp[1] = stamp[2] = global_ns();
      } else if (ph.kind != kPhaseGemv) {
        const int SP = P.attn_split;
        if (cta < P.head_num * SP) {
          if (ph.kind == kPhaseAttnFlash)
            pipe = attention_flash_phase<KV>(P, cta / SP, cta % SP, pos, pipe, hand_tag(ph.hand_in), hand_tag(ph.hand_out), stamp);
          else if (ph.kind == kPhaseAttnFused)
            pipe = attention_fused_phase(P, cta, pos, pipe, hand_tag(ph.hand_in), hand_tag(ph.hand_out), stamp);
          else if (ph.kind == kPhaseAttention)
            pipe = attention_scores_phase(P, cta / SP, cta % SP, pos, pipe, hand_tag(ph.hand_in), hand_tag(ph.hand_out), stamp);
          else
            pipe = attention_pv_phase(P, cta / SP, cta % SP, pos, pipe, hand_tag(ph.hand_in), hand_tag(ph.hand_aux),
                                          hand_tag(ph.hand_out), stamp);
        }
        if (stamp) stamp[1] = stamp[2] = global_ns();
      } else if (!(ph.cls && tok < P.skip_cls_tokens)) {
        // A prompt token (llama3.cpp:733-745: predict(..., is_prompt = true) discards the logits and
        // returns -1) skips the classifier -- its weights are not even streamed -- but keeps the grid
        // barrier that closes the token.
        const Carry out = gemv_phase<F, KV, LP, PROF>(P, Carry{pipe, best.v, best.i}, tok, pos, emb_row, stamp);
        pipe = out.pipe;
        best.v = out.best_v, best.i = out.best_i;
      }
      if (stamp && pi + 1 < P.n_phases) stamp[3] = global_ns();  // no barrier closes a phase but the last
    }
    // The token's one grid barrier: the classifier's logits and argmax partials (or the gather's) are complete
    // behind it, and so are the K/V rows of this token that the producer streams for the next one.
    grid_barrier(P.barrier, bar_target, G);
    if (stamp) stamp[3] = global_ns();

    // ---- the id: every CTA folds the per-CTA partials identically, or with top-k or top-p draws it itself ----
    int next;
    if (LP && !(tok < P.skip_cls_tokens)) {
      next = draw_with_logprobs(P, pos, step);
    } else if (!(tok < P.skip_cls_tokens) && sampling::needs_draw(*P.sampling, P.vocab_size)) {
      next = draw_truncated(P, pos);
    } else {
      next = fold_cta_partials(P);
    }
    // Every CTA (and every tensor-parallel rank) holds the same `next`, so the stop needs no exchange.
    bool stop = false;
#pragma unroll
    for (int i = 0; i < kMaxStopIds; ++i) stop |= P.stop_ids[i] == next;
    if (cta == 0 && tid == 0) {
      if (P.out_tokens != nullptr && step < P.max_steps) P.out_tokens[step] = next;
      if (P.stream_ids != nullptr) {  // the id, then (release, system scope) the count the host polls
        P.stream_ids[step] = next;
        st_release_sys(P.stream_count, step + 1);
      }
    }
    token = (P.teacher != nullptr && step + 1 < P.max_steps) ? P.teacher[step + 1] : next;
    if (!stop && tok + 1 < P.n_tokens) record_fed(P, pos + 1, token);  // the next token of this launch
    if (static_cast<unsigned>(token) >= static_cast<unsigned>(P.vocab_size)) token = 0;
    pos += 1;
    step += 1;
    if (cta == 0 && tid == 0 && (tok == P.n_tokens - 1 || stop)) {
      P.state->token = token;
      P.state->pos = pos;
      P.state->step = step;
      P.state->next = next;
    }
    if (stop) {
      // The producer may have issued stages of the next token already, and may be waiting for a slot that
      // will never be freed.  Tell it to stop, then wait until every fill it issued has landed: the CTA may
      // not exit with a bulk copy into its shared memory in flight.
      if (tid == 0) g_stop = 1;
      unsigned end;
      while ((end = g_prod_end) == 0u) {
      }
      const Pipe last{static_cast<int>((end - 1u) >> 1), (end - 1u) & 1u};
      while (pipe.slot != last.slot || pipe.parity != last.parity) {
        mbar_wait(&full_bar[pipe.slot], pipe.parity);
        pipe.advance(S);
      }
      return;
    }
  }
}

template <WeightFormat F, int KV, bool LP, bool PROF>
__global__ void __launch_bounds__(kConsumerThreads + 32, 1) decode_megakernel(const __grid_constant__ Params P) {
  megakernel_body<F, KV, LP, PROF>(P);
}

}  // namespace mega

// ================================== host side ======================================================
using mega::Params;
using mega::Phase;

namespace {
template <typename K>
const void* fn(K* kernel) {
  return reinterpret_cast<const void*>(kernel);
}
// The instantiations that run a model of weight format F over a cache of element KV (a kllm_decoder_desc::kv_cache
// value): the plain one, the profiling one kllm_decoder_profile launches (null where there is none: a bf16 or fp8
// cache, or bf16 weights) and the log-probability one.
struct Kernels {
  const void *plain, *prof, *lp;
};
template <WeightFormat F, int KV>
Kernels kernels_for() {
  using mega::decode_megakernel;
  const void* prof = nullptr;
  if constexpr (F != WeightFormat::kBf16 && KV == KLLM_KV_F32) prof = fn(decode_megakernel<F, KV, false, true>);
  return Kernels{fn(decode_megakernel<F, KV, false, false>), prof, fn(decode_megakernel<F, KV, true, false>)};
}
template <WeightFormat F>
Kernels kernels_for(int kv) {
  switch (kv) {
    case KLLM_KV_BF16: return kernels_for<F, KLLM_KV_BF16>();
    case KLLM_KV_FP8: return kernels_for<F, KLLM_KV_FP8>();
    default: return kernels_for<F, KLLM_KV_F32>();
  }
}
Kernels kernels_for(WeightFormat f, int kv) {
  switch (f) {
    case WeightFormat::kInt8: return kernels_for<WeightFormat::kInt8>(kv);
    case WeightFormat::kBf16: return kernels_for<WeightFormat::kBf16>(kv);
    default: return kernels_for<WeightFormat::kF32>(kv);
  }
}
constexpr int kThreads = mega::kConsumerThreads + 32;  // the consumer warps and the ring producer
// Ring stage of bf16 weights, per numerics mode as fp32's.  H100 80GB HBM3, 700 W, tok/s at positions 1 / 512 / 2047
// (tools/bench_weights.py, DESIGN.md 5.11), 16 / 24 / 32 KB:
//   exact: TinyLlama-1.1B at 2047 607 / 710 / 745, Qwen2.5-0.5B at 2047 703 / 799 / 848 -- the exact attention's
//          tiles shrink with the stage; Llama-2-7B within 2-6 % of each other.  32 KB.
//   fast:  24 KB is at or above 32 KB at every measured point of the three models (TinyLlama-1.1B +1-2 %,
//          Qwen2.5-0.5B +2-7 %, Llama-2-7B +1 %); 16 KB is best on Llama-2-7B (+4-5 % over 24 KB) but loses 2-6 % on
//          TinyLlama-1.1B.  24 KB.
constexpr int kW16StageBytes = 32 * 1024;
constexpr int kW16FastStageBytes = 24 * 1024;
}  // namespace

// In order: decide the geometry and every refusal, then allocate the scratch block, then fill it and the launch
// parameters.  Nothing after the allocation refuses.
int MegaEngine::init(const DecoderModel& dm, const MegaModel& m, cudaStream_t stream) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return KLLM_E_NODEVICE;
  int sms = 0, coop = 0, max_smem = 0;
  KLLM_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  KLLM_TRY(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  KLLM_TRY(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  if (!coop) return KLLM_E_UNSUPPORTED;

  const int dim = dm.dim, hid = dm.hidden_dim, hs = dm.head_size, kvd = dm.kv_dim, q_rows = dm.q_rows;
  const bool int8 = dm.format == WeightFormat::kInt8;
  const bool w16 = dm.format == WeightFormat::kBf16;  // 2-byte rows through the same ring
  const int wb = weight_bytes(dm.format);
  // One CTA per SM, but never more CTAs than the shortest row-parallel phase has rows: the
  // slot-reuse argument of the tagged hand-offs wants every CTA to own rows in every producing
  // phase (a CTA without rows gates nothing and could be overtaken).  Small test shapes only.
  const int grid = std::min(sms, std::min(dim, hid));
  if (grid < dm.head_num) return KLLM_E_UNSUPPORTED;  // attention: one CTA per (local) query head
  // shapes the ring handles: 16-byte rows, 128-byte aligned kv rows (L1-cached reads stay exact);
  // head_size <= 128: the K-tile producer issues one bulk copy per lane for hs/4 <= 32 chunk columns
  if ((dim & 3) || (hid & 3) || (q_rows & 3) || (hs & 3) || hs > 128) return KLLM_E_UNSUPPORTED;
  if (int8 && ((dim & 15) || (hid & 15) || (q_rows & 15) || (dm.group_size & 3))) return KLLM_E_UNSUPPORTED;
  if (w16 && ((dim & 7) || (hid & 7) || (q_rows & 7))) return KLLM_E_UNSUPPORTED;  // bf16 rows: 16-byte multiples
  if ((hs * 4) % 16 != 0) return KLLM_E_UNSUPPORTED;
  if (int8) {
    const int dims[3] = {dim, hid, q_rows};
    for (int d : dims)
      if (d % dm.group_size != 0 || ((d / dm.group_size) * 4) % 16 != 0) return KLLM_E_UNSUPPORTED;
  }
  // int8 arithmetic: "exact" reproduces the reference's fma(x * scale, float(w), acc) per element bit for
  // bit; "fast" is the dp4a fixed-point mode (toleranced, ~3.5x fewer instructions)
  // The same switch frees the attention's summation order (flash-decoding, attention_flash_phase).
  // kllm_decoder_desc::numerics picks the mode; KLLM_MODE=exact|fast overrides.
  int fast = m.numerics == 1 ? 1 : 0;
  if (const char* e = getenv("KLLM_MODE")) fast = std::string(e) == "fast" ? 1 : 0;
  // bf16 and fp8 KV caches: toleranced variants of the flash attention only, over 16-byte chunks of 8 (bf16) or 16
  // (fp8) dims with a quarter of the head per lane (head_size % 32 == 0, % 64 == 0); refused rather than run in any
  // other form
  const int kv = m.kv_cache;
  if (kv != KLLM_KV_F32 && kv != KLLM_KV_BF16 && kv != KLLM_KV_FP8) return KLLM_E_INVALID;
  const int kv_esz = prefill::kv_elem_bytes(kv);  // bytes per cached element
  if (kv != KLLM_KV_F32 && (!fast || m.tp_world > 1 || hs % (64 / kv_esz) != 0)) return KLLM_E_UNSUPPORTED;
  if (kv == KLLM_KV_FP8 && m.kv_scales == nullptr) return KLLM_E_INVALID;
  const Kernels ks = kernels_for(dm.format, kv);

  // The residual exchange after o_proj and down_proj is tagged (under tensor parallelism it IS the
  // all-reduce), and so are the hand-offs q|k|v -> attention -> Wo and SwiGLU -> W2: the one grid
  // barrier of a token follows its last phase.
  const int W = m.tp_world > 1 ? m.tp_world : 1;
  if (W != 1 && W != 2 && W != 4 && W != 8) return KLLM_E_UNSUPPORTED;

  // ---- shared memory plan -----------------------------------------------------------------------
  const int max_in = std::max(std::max(dim, hid), q_rows);
  int xbuf = max_in * 4;
  const int attn_ws = 2 * hs * 4;
  xbuf = std::max(xbuf, attn_ws);
  // Stage size: whole rows, so pick it to waste little of the ring on the model's row lengths.
  // fp32: 32 KB (4 rows of dim 2048, 2 of 4096).  int8: 27 KB = 6 rows of dim 4096 (+ scales) or
  // 2 rows of hidden 11008, which leaves six stages next to the 44 KB input vector and the 16 KB
  // residual stream of Llama-2-7B.
  // fp32 in the fast numerics (fp32 cache), when a 16 KB stage still holds two input rows of dim (dim <= 2048): 12 ×
  // 16 KB.  The same ring in twice the slots is released at half the grain: a stage of 2 rows of dim 2048 is one
  // task of one warp, so all 8 warps drain the ring at once instead of 6, and TinyLlama's W2 (22.5 KB rows, 2 chunks
  // of 12 and 10 KB) fills it as well as one row filled 32 KB.  H100 80GB HBM3, 700 W: TinyLlama-1.1B 670 tok/s
  // against 627 with 32 KB (20 KB: 649, 24 KB: 645), Qwen2.5-0.5B 1058 against 1032.  At dim 4096 a 16 KB stage is
  // ONE row, a task no longer shares its x loads, and Llama-2-7B fell from 108 to 80 tok/s.  The flash tiles shrink
  // with the stage (head_size 64: 64 timesteps).
  const bool small_stages = fast && kv == KLLM_KV_F32 && !w16 && 2 * dim * 4 <= 16 * 1024;
  int stage_bytes = int8 ? 27 * 1024 : w16 ? (fast ? kW16FastStageBytes : kW16StageBytes) : small_stages ? 16 * 1024
                                                                                                : 32 * 1024;
  if (const char* e = getenv("KLLM_STAGE_BYTES")) stage_bytes = atoi(e);
  stage_bytes = (stage_bytes + 127) & ~127;
  const int attn_tile = std::min(stage_bytes / (hs * kv_esz), mega::kConsumerThreads) & ~31;  // a timestep per thread
  if (attn_tile < 32) return KLLM_E_UNSUPPORTED;
  if (fast) {  // flash attention: a lane quartet per timestep, warp partials (m, l, o[hs]) in the input buffer
    if (hs & 15) return KLLM_E_UNSUPPORTED;
    xbuf = std::max(xbuf, (2 * hs + mega::kConsumerWarps * (hs + 2)) * 4);
  }
  // the top-k / top-p draw's scratch after the classifier (draw_truncated): the histogram and at least 64 candidates
  xbuf = std::max(xbuf, sampling::kDrawScratchBase + 64 * 8);
  // ... and the log-probabilities' (logprob_partial, logprob_record): the top-N select keeps one maximum per thread
  xbuf = std::max(xbuf, sampling::logprob_scratch_bytes(mega::kConsumerThreads));
  xbuf = (xbuf + 127) & ~127;
  const int xres = (dim * 4 + 127) & ~127;  // the CTA's copy of the residual stream
  const int budget = max_smem - xbuf - xres - 3584;  // static shared memory (1.1 KB) + slack
  int stages = budget / stage_bytes;
  if (stages > mega::kMaxStages) stages = mega::kMaxStages;
  if (stages < 2) return KLLM_E_UNSUPPORTED;
  // attention split: SP CTAs per query head (power of two, <= 8), each owning head_size / SP output dims
  // (a multiple of 4 floats so that V slice rows stay 16-byte units for the bulk copies)
  if (dm.seq_len & 3) return KLLM_E_UNSUPPORTED;
  int split = 1;
  while (split * 2 <= 8 && dm.head_num * split * 2 <= grid && (hs / (split * 2)) % 4 == 0 && hs % (split * 2) == 0)
    split *= 2;
  int split_cap = split;
  // The split costs one more hand-off per layer: worth it when a head's K and V are big
  // (head_size 128: 1 MB per head at context 1024), not for head_size 64.
  if (hs < 128) split = 1;
  if (fast) {  // flash: split by timestep, any power of two whose partial triples fit the scores area
    split = 1;
    while (split * 2 <= 8 && dm.head_num * split * 2 <= grid && split * 2 * (hs + 2) <= dm.seq_len) split *= 2;
    split_cap = split;
  }
  if (const char* e = getenv("KLLM_ATTN_SPLIT")) {
    const int v = atoi(e);
    if (v >= 1 && v <= split_cap && (v & (v - 1)) == 0) split = v;
  }
  const int vsplit = fast ? 1 : split;
  const int attn_tile_v = (stage_bytes / ((hs / vsplit) * kv_esz)) & ~31;
  if (attn_tile_v < 32) return KLLM_E_UNSUPPORTED;
  const size_t smem_bytes = static_cast<size_t>(xbuf) + xres + static_cast<size_t>(stages) * stage_bytes;

  // ---- the ring plan of every GEMV phase ----------------------------------------------------------------
  auto plan = [&](Phase& p) -> int {
    const int row_bytes = p.in_dim * wb;
    p.group_size = dm.group_size;
    p.group_shift = dm.group_shift;
    if (int8) p.scale_row_bytes = (p.in_dim / dm.group_size) * 4;
    const int rpu = p.swiglu ? 2 : 1;
    const int per_row = row_bytes + p.scale_row_bytes;
    if (per_row * rpu <= stage_bytes) {
      int rows = stage_bytes / per_row;
      rows -= rows % rpu;
      rows = std::min(rows, 32);  // one bulk copy per producer lane
      p.rows_per_stage = rows;
      p.chunks_per_row = 1;
      p.chunk_elems = p.in_dim;
      p.scale_off = ((rows * row_bytes) + 127) & ~127;
      if (p.scale_off + rows * p.scale_row_bytes > stage_bytes) {
        // shrink until weights + scales fit
        while (rows > rpu && (((rows * row_bytes + 127) & ~127) + rows * p.scale_row_bytes) > stage_bytes)
          rows -= rpu;
        p.rows_per_stage = rows;
        p.scale_off = ((rows * row_bytes) + 127) & ~127;
      }
    } else {
      if (int8 || p.swiglu) return KLLM_E_UNSUPPORTED;
      const int chunk_max = (stage_bytes / wb) & ~511;  // elements: a multiple of 128 packs
      p.chunks_per_row = (p.in_dim + chunk_max - 1) / chunk_max;
      int ce = (p.in_dim + p.chunks_per_row - 1) / p.chunks_per_row;
      ce = (ce + 511) & ~511;
      p.chunk_elems = ce;
      p.chunks_per_row = (p.in_dim + ce - 1) / ce;
      p.rows_per_stage = 1;
      p.scale_off = 0;
    }
    return 0;
  };
  // The plan depends only on the input length and the SwiGLU pairing: one per GEMV of the table, decided here.
  Phase qkv{}, wo{}, ffn{}, w2{}, cls{};
  qkv.in_dim = dim, wo.in_dim = q_rows, ffn.in_dim = dim, ffn.swiglu = 1, w2.in_dim = hid, cls.in_dim = dim;
  for (Phase* p : {&qkv, &wo, &ffn, &w2, &cls})
    if (int rc = plan(*p)) return rc;
  // Tensor parallel: shard the classifier by vocabulary when the exchange area can carry a rank's
  // rows (kllm_comm_create(max_count >= vocab / world)); every rank still holds the whole matrix and
  // reads only its rows.  Otherwise it stays replicated.
  const int V = dm.vocab_size;
  const bool shard = W > 1 && V % W == 0 && m.tp_stride >= V / W;
  const int cls_rows = shard ? V / W : V;

  // process-wide and only ever raised: another decoder's engine launches the same instantiations at its own size
  for (const void* k : {ks.plain, ks.prof, ks.lp})
    if (k != nullptr)
      if (int rc = smem_opt_in(k, smem_bytes)) return rc;
  int occ_lp = 0;
  KLLM_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_lp, ks.lp, kThreads, smem_bytes));
  if (occ_lp < 1) return KLLM_E_UNSUPPORTED;
  int occ = 0;
  KLLM_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, ks.plain, kThreads, smem_bytes));
  if (occ < 1) return KLLM_E_UNSUPPORTED;

  // ---- the scratch block: one allocation, each part at a 256-byte aligned offset -------------------------
  // per layer QKV, the attention (one phase, or the split's two), Wo, W1|W3 and W2; then the classifier
  const int n_phases = dm.layer_num * ((fast || split == 1) ? 5 : 6) + (shard ? 2 : 1);
  size_t bytes = 0;
  auto part = [&bytes](size_t n) {
    const size_t off = bytes;
    bytes += (n + 255) & ~static_cast<size_t>(255);
    return off;
  };
  using u64 = unsigned long long;
  const size_t hand_off = part(sizeof(u64) * (2 * q_rows + 2 * kvd + hid));  // q | raw k | v | attention | h
  const size_t scores_off = part(sizeof(u64) * dm.head_num * dm.seq_len);    // tagged scores of the split attention
  // the split P.V phase's probabilities past shared memory, one row per CTA
  const size_t probs_off = part(fast || split == 1 ? 0 : sizeof(float) * dm.head_num * split * dm.seq_len);
  const size_t tagged_off = part(W == 1 ? sizeof(u64) * 2 * dim : 0);       // single-GPU exchange area
  const size_t phases_off = part(sizeof(Phase) * n_phases);
  const size_t barrier_off = part(128);
  const size_t arg_val_off = part(sizeof(float) * grid), arg_idx_off = part(sizeof(int) * grid);
  // lp_part [grid] float2, then lp_cand_v / lp_cand_i [grid][kMaxTopLogprobs]
  const size_t lp_off = part(static_cast<size_t>(grid) * (sizeof(float2) + 8 * sampling::kMaxTopLogprobs));
  KLLM_TRY(cudaMalloc(&scratch_, bytes));
  unsigned char* const s = static_cast<unsigned char*>(scratch_);
  u64 *t_q = reinterpret_cast<u64*>(s + hand_off), *t_k = t_q + q_rows, *t_v = t_k + kvd, *t_attn = t_v + kvd,
      *t_h = t_attn + q_rows;

  // ---- phase table ---------------------------------------------------------------------------------
  std::vector<Phase> ph;
  int hands = 0;
  int exch = 0;
  // a phase whose input is the residual stream: x_old (shared memory) + partials of the last exchange;
  // before the first exchange (layer 0's QKV) the stream is the embedding row
  auto input_is_x = [&](Phase& p) {
    if (exch == 0) return;
    p.tp_in = 1;
    p.exch = exch - 1;
  };

  // a GEMV segment of `rows` rows of the matrix `w`
  auto seg = [](const Matrix& w, float* out, int rows, int head_major = 0, unsigned long long* tag_out = nullptr) {
    return mega::Seg{w.w, w.scales, w.bias, out, 0, rows, head_major, tag_out};
  };
  for (int l = 0; l < dm.layer_num; ++l) {
    const LayerWeights& lw = dm.layers[l];
    const size_t layer_off = static_cast<size_t>(l) * dm.seq_len * kvd;
    {  // attention_rms + q | k | v (+bias).  q and the raw k are handed off only; v also goes into the cache.
      Phase p = qkv;
      p.kind = mega::kPhaseGemv;
      p.n_seg = 3;
      input_is_x(p);
      p.norm_w = lw.attn_norm;
      p.norm_eps = dm.eps;
      p.seg[0] = seg(lw.q, nullptr, q_rows, 0, t_q);
      p.seg[1] = seg(lw.k, nullptr, kvd, 0, t_k);
      // the bf16 and fp8 caches' instantiations store bf16 or fp8 elements in the epilogue
      float* vrows = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(m.value_cache) + layer_off * kv_esz);
      p.seg[2] = seg(lw.v, vrows, kvd, 1, t_v);
      p.layer = l;  // the fp8 cache's value epilogue reads its layer's scales
      p.units = q_rows + 2 * kvd;
      p.hand_out = hands;
      ph.push_back(p);
    }
    if (fast || split == 1) {  // flash-decoding (`split` CTAs per head by timestep) or fused: one phase
      Phase p{};
      p.kind = fast ? mega::kPhaseAttnFlash : mega::kPhaseAttnFused;
      p.layer = l;
      p.tq = t_q, p.tk = t_k, p.tv = t_v, p.ta = t_attn;
      p.hand_in = hands++;
      p.hand_out = hands;
      ph.push_back(p);
    } else {
      int qkv_hand = 0;
      {  // attention, scores: CTA (head, s) scores the K tiles s, s + SP, ... and publishes them tagged
        Phase p{};
        p.kind = mega::kPhaseAttention;
        p.layer = l;
        p.tq = t_q, p.tk = t_k, p.tv = t_v;
        p.hand_in = hands++;
        qkv_hand = p.hand_in;
        p.hand_out = hands;
        ph.push_back(p);
      }
      {  // attention, softmax + P.V: CTA (head, s) owns output dims [s dv, (s + 1) dv)
        Phase p{};
        p.kind = mega::kPhaseAttnPV;
        p.layer = l;
        p.hand_in = hands++;
        p.tv = t_v, p.ta = t_attn;
        p.hand_aux = qkv_hand;
        p.hand_out = hands;
        ph.push_back(p);
      }
    }
    {  // wo, added to the residual stream by the readers of the exchange (llama3.cpp:672-684)
      Phase p = wo;
      p.kind = mega::kPhaseGemv;
      p.n_seg = 1;
      p.tag_in = t_attn;
      p.hand_in = hands++;
      p.seg[0] = seg(lw.o, nullptr, dim);
      p.units = dim;
      p.tp_out = 1;
      p.exch_out = exch++;
      ph.push_back(p);
    }
    {  // ffn rmsnorm + w1 | w3 -> swiglu (llama3.cpp:686-708)
      Phase p = ffn;
      p.kind = mega::kPhaseGemv;
      p.n_seg = 2;
      input_is_x(p);
      p.norm_w = lw.ffn_norm;
      p.norm_eps = dm.eps;
      p.seg[0] = seg(lw.w1, nullptr, hid, 0, t_h);
      p.seg[1] = seg(lw.w3, nullptr, hid);
      p.units = hid;
      p.hand_out = hands;
      ph.push_back(p);
    }
    {  // w2, added to the residual stream by the readers of the exchange (llama3.cpp:711-719)
      Phase p = w2;
      p.kind = mega::kPhaseGemv;
      p.n_seg = 1;
      p.tag_in = t_h;
      p.hand_in = hands++;
      p.seg[0] = seg(lw.w2, nullptr, dim);
      p.units = dim;
      p.tp_out = 1;
      p.exch_out = exch++;
      ph.push_back(p);
    }
  }
  {  // final rmsnorm + classifier (+ argmax partials)
    Phase p = cls;
    p.kind = mega::kPhaseGemv;
    p.n_seg = 1;
    input_is_x(p);
    p.norm_w = dm.final_norm;
    p.norm_eps = dm.eps;
    p.cls = 1;
    if (shard) {
      p.seg[0] = seg(dm.rows_from(dm.cls, static_cast<size_t>(m.tp_rank) * cls_rows, dim), nullptr, cls_rows);
      p.units = cls_rows;
      p.tp_out = 1;  // rows go to every rank's exchange area as tagged words
      p.exch_out = exch++;
      ph.push_back(p);
      Phase g{};
      g.kind = mega::kPhaseGather;
      g.cls = 1;
      g.argmax = 1;
      g.units = V;
      g.in_dim = cls_rows;
      g.exch = p.exch_out;
      g.seg[0].out = m.logits;
      ph.push_back(g);
    } else {
      p.seg[0] = seg(dm.cls, m.logits, V);
      p.units = V;
      p.argmax = 1;
      ph.push_back(p);
    }
  }

  // zeroed: the hand-off words, the score words and the exchange area carry tag 0, the barrier word counts from 0
  KLLM_TRY(cudaMemsetAsync(s, 0, bytes, stream));
  KLLM_TRY(cudaMemcpyAsync(s + phases_off, ph.data(), sizeof(Phase) * n_phases, cudaMemcpyHostToDevice, stream));
  KLLM_TRY(cudaStreamSynchronize(stream));  // ph (host vector) must outlive the async copy

  Params P{};
  P.phases = reinterpret_cast<const Phase*>(s + phases_off);
  P.n_phases = n_phases;
  P.n_cls_phases = shard ? 2 : 1;
  P.int8_fast = (int8 && fast) ? 1 : 0;
  P.num_stages = stages;
  P.stage_bytes = stage_bytes;
  P.xbuf_bytes = xbuf;
  P.xres_bytes = xres;
  P.attn_tile = attn_tile;
  P.attn_tile_v = attn_tile_v;
  P.attn_split = split;
  P.attn_vsplit = vsplit;
  P.scores = reinterpret_cast<u64*>(s + scores_off);
  P.group_size = dm.group_size;
  P.dim = dm.dim;
  P.vocab_size = dm.vocab_size;
  P.head_num = dm.head_num;
  P.head_size = dm.head_size;
  P.kv_dim = dm.kv_dim;
  P.kv_mul = dm.kv_mul;
  P.seq_len = dm.seq_len;
  P.flavour = dm.flavour;
  P.tok_emb = dm.tok_emb;
  P.score = m.score;
  P.probs = reinterpret_cast<float*>(s + probs_off);
  P.key_cache = m.key_cache;
  P.value_cache = m.value_cache;
  P.sin_cache = m.sin_cache;
  P.cos_cache = m.cos_cache;
  P.state = m.state;
  P.out_tokens = m.out_tokens;
  P.max_steps = dm.seq_len;
  P.barrier = reinterpret_cast<unsigned*>(s + barrier_off);
  P.tp_world = W;
  P.tp_rank = W > 1 ? m.tp_rank : 0;
  P.tp_stride = W > 1 ? m.tp_stride : dim;
  for (int r = 0; r < 8; ++r) P.tp_data[r] = W > 1 ? m.tp_data[r] : nullptr;
  if (W == 1) P.tp_data[0] = reinterpret_cast<u64*>(s + tagged_off);
  P.exch_per_token = exch;
  P.hands_per_token = hands;
  P.arg_val = reinterpret_cast<float*>(s + arg_val_off);
  P.arg_idx = reinterpret_cast<int*>(s + arg_idx_off);
  P.sampling = m.sampling;
  P.logits = m.logits;
  P.hist = m.hist;
  P.penalized = m.penalized;
  P.prof_token = -1;
  for (int i = 0; i < mega::kMaxStopIds; ++i) P.stop_ids[i] = -1;  // ids are >= 0: no stop
  P.lp_part = reinterpret_cast<float2*>(s + lp_off);
  P.lp_cand_v = reinterpret_cast<float*>(P.lp_part + grid);
  P.lp_cand_i = reinterpret_cast<int*>(P.lp_cand_v + static_cast<size_t>(grid) * sampling::kMaxTopLogprobs);
  P.lp_rec = m.lp_rec;
  if (kv == KLLM_KV_FP8) {
    const size_t n = static_cast<size_t>(dm.layer_num) * dm.kv_head_num;
    P.kv_scale_k = m.kv_scales, P.kv_scale_v = m.kv_scales + n;
    P.kv_inv_k = m.kv_scales + 2 * n, P.kv_inv_v = m.kv_scales + 3 * n;
  }
  base_ = P;
  stream_ = stream;
  grid_ = grid;
  fast_ = fast;
  cls_rows_ = cls_rows;
  kernel_ = ks.plain, kernel_prof_ = ks.prof, kernel_lp_ = ks.lp;
  smem_bytes_ = smem_bytes;
  ready_ = true;
  return 0;
}

int MegaEngine::destroy() {
  const cudaError_t e = cudaFree(scratch_);  // a null pointer frees nothing
  scratch_ = nullptr;
  ready_ = false;
  return static_cast<int>(e);
}

// base_ with the settings of this launch and the tag and barrier bases the tokens before it left
Params MegaEngine::params(const DrawSettings& cfg, int n_tokens) const {
  Params P = base_;
  P.n_tokens = n_tokens;
  P.penalty = cfg.penalty;
  P.lp_top_n = cfg.lp_top_n;
  P.barrier_base = barrier_base_;
  P.tp_seq_base = tp_seq_base_;
  P.hand_base = hand_base_;
  return P;
}

int MegaEngine::launch(const Params& P) {
  void* args[] = {const_cast<Params*>(&P)};
  // the profiling instantiation records no log-probabilities; the LP one runs while they are on
  const void* k = P.prof != nullptr ? kernel_prof_ : P.lp_top_n >= 0 ? kernel_lp_ : kernel_;
  if (k == nullptr) return KLLM_E_UNSUPPORTED;
  KLLM_TRY(cudaLaunchCooperativeKernel(const_cast<void*>(k), dim3(grid_), dim3(kThreads), args, smem_bytes_, stream_));
  count_launch();
  return 0;
}

// The tags and barrier counts the next launch waits for continue from where the tokens that ran left them.
void MegaEngine::account(int n_tokens) {
  tp_seq_base_ += static_cast<unsigned>(n_tokens) * static_cast<unsigned>(base_.exch_per_token);
  hand_base_ += static_cast<unsigned>(n_tokens) * static_cast<unsigned>(base_.hands_per_token);
  barrier_base_ += static_cast<unsigned>(n_tokens) * static_cast<unsigned>(grid_);  // one grid barrier per token
}

int MegaEngine::run(const DrawSettings& cfg, int n_tokens, const int32_t* teacher_dev, unsigned long long* prof_dev,
                    int prof_token, int skip_cls_tokens, int lp_target) {
  if (!ready_) return KLLM_E_STATE;
  Params P = params(cfg, n_tokens);
  P.teacher = teacher_dev;
  P.prof = prof_dev;
  P.prof_token = prof_token;
  P.skip_cls_tokens = skip_cls_tokens;
  P.lp_target = lp_target;
  if (int rc = launch(P)) return rc;
  account(n_tokens);
  return 0;
}

int MegaEngine::run_until(const DrawSettings& cfg, int n_tokens, const int32_t* stop_ids, int n_stop,
                          int32_t* stream_ids, int32_t* stream_count) {
  if (!ready_) return KLLM_E_STATE;
  if (n_stop < 0 || n_stop > mega::kMaxStopIds) return KLLM_E_INVALID;
  Params P = params(cfg, n_tokens);
  for (int i = 0; i < n_stop; ++i) P.stop_ids[i] = stop_ids[i];
  P.stream_ids = stream_ids;
  P.stream_count = stream_count;
  return launch(P);
}

}  // namespace kllm
