// Batched GEMM for prompt prefill on the Hopper tensor cores (sm_90a):
//     out[T, N] = x[T, K] . w[N, K]^T        fp32 storage, TF32 multiply, fp32 accumulate in registers
// for fp32 weights (kllm_gemm_tf32) and for int8 group-quantised weights (kllm_gemm_w8_tf32), where
// w[n, k] = scales[(n K + k) / group_size] * q[n, k] is dequantised into the shared-memory tile.
//
// The reference feeds a prompt through one full single-token forward per position (demo/main.cpp:
// 18-23, llama3.cpp:147-167) -- T GEMVs that stream every weight T times.  With the T prompt rows
// as the N dimension of a wgmma the weights are streamed once per 256 tokens.
//
// This is an explicitly TOLERANCED kernel: TF32 keeps 10 mantissa bits of each operand, so results
// agree with the fp32 GEMV path to ~1e-3 relative, not bit for bit (tests/test_prefill_gpu.py states
// the bound).  The bit-exact decode path never calls it.
//
// Structure (one CTA per 128 weight rows x one block of BN tokens, three warpgroups):
//   warpgroup 0    TMA producer (one thread): cp.async.bulk.tensor 2-D tiles of w [128 x 32 fp32] and
//                  x [BN x 32 fp32], 128-byte swizzle, into a 4-stage shared-memory ring (SASS: UTMALDG)
//   warpgroups 1-2 consumers, 64 weight rows each: round the stage's operands to the nearest tf32 in place,
//                  then 4 x wgmma.mma_async m64nBNk8 tf32 per stage, both
//                  operands from shared memory, accumulators in registers (SASS: HGMMA); a stage is
//                  released once the wgmma group after it has been issued and the one reading it retired
//   epilogue       each consumer thread stores its accumulator fragment straight to out
//
// int8 weights (template parameter F = WeightFormat::kInt8): the producer loads the weight tile as bytes [128 x 32 int8] into
// a 4 KB staging area of the stage; each consumer warpgroup dequantises its 64 rows (scale * q in fp32,
// rounded to the nearest tf32) into the same 128-byte-swizzled fp32 A tile TMA would have written, so the
// wgmma descriptors and instructions are the fp32 path's.  The scale of a row is constant over a 32-column
// K block (group_size % 32 == 0, in_dim % group_size == 0) and is read with an ordinary non-coherent load
// one K block ahead: scale rows can be 4 bytes, which TMA cannot copy.  A stage is dequantised while the
// wgmma group of the stage before it is still running.
//
// bf16 weights (F = WeightFormat::kBf16, kllm_gemm_bf16_tf32): the same staging with a [128 x 32 bf16] tile of
// 64-byte rows, widened into the fp32 A tile.  A bf16 value widens exactly and is already a tf32 value, so the A
// tile holds what kllm_gemm_tf32 holds after its rounding of the widened weights: the results are bit-identical.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/kllm_b200.h"
#include "kllm_host.h"

namespace kllm {
namespace tc {

constexpr int BM = 128;     // weight rows per CTA = 2 consumer warpgroups x wgmma M 64
constexpr int BK = 32;      // fp32 elements per K block = 128 bytes = one swizzle-128B row
constexpr int WG_K = 8;     // tf32: 32 bytes of K per wgmma
constexpr int STAGES = 4;
constexpr int A_BYTES = BM * BK * 4;  // 16 KB
// bytes of the weight staging area per stage: the int8 (4 KB, rows of 32 bytes) or bf16 (8 KB, rows of 64 bytes)
// weight tile as loaded; fp32 tiles land in the A tile directly
__host__ __device__ constexpr int staging_bytes(WeightFormat f) {
  return f == WeightFormat::kF32 ? 0 : BM * BK * weight_bytes(f);
}
constexpr int THREADS = 384;

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n .reg .pred p;\n WAIT_%=:\n"
      " mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      " @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Shared-memory matrix descriptor of a K-major tile with 128-byte swizzle (PTX ISA, "Matrix Descriptor
// Format" of wgmma): start address >> 4 in bits [0,14), leading byte offset (unused with swizzle; 1) in
// [16,30), stride byte offset = 8 rows x 128 B = 1024 B >> 4 in [32,46), base offset 0 (tiles are
// 1024-byte aligned), swizzle mode 128B = 1 in [62,64).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
  return static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// D[64 x N] (+)= A[64 x 8] . B[N x 8]^T, tf32 operands from shared memory, fp32 accumulators: thread t of the
// warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 j + 2 (t % 4) (+ 1), d[4 j .. 4 j + 3].
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n"
      " wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n"
      " wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
      " wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_tf32<256>(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %130, 0;\n"
      " wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1;\n}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// n float4 of shared memory rounded to the nearest tf32 (ties away from zero) by the 128 threads of a warpgroup
__device__ __forceinline__ void round_tf32(float4* p, int n, int t) {
  for (int i = t; i < n; i += 128) {
    float4 v = p[i];
    float* e = reinterpret_cast<float*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint32_t r;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(e[j]));
      e[j] = __uint_as_float(r);
    }
    p[i] = v;
  }
}

// Thread (r, half) of a consumer warpgroup turns the 16 int8 weights of columns 16 half .. + 15 of its local
// row r into scale * q rounded to the nearest tf32, and stores them as four 16-byte chunks of the row in the
// 128-byte swizzle TMA uses: chunk c of row r lives at r * 128 + (c ^ (r & 7)) * 16.
__device__ __forceinline__ void dequant_w8(const uint8_t* src, uint8_t* a_rows, int r, int half, float scale) {
  const int4 q = *reinterpret_cast<const int4*>(src);
  const int words[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float e[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float v = scale * static_cast<float>(static_cast<int8_t>((words[j] >> (8 * i)) & 0xff));
      uint32_t u;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
      e[i] = __uint_as_float(u);
    }
    const int c = 4 * half + j;
    *reinterpret_cast<float4*>(a_rows + r * 128 + ((c ^ (r & 7)) << 4)) = make_float4(e[0], e[1], e[2], e[3]);
  }
}

// Thread (r, half) of a consumer warpgroup widens the 16 bf16 weights of columns 16 half .. + 15 of its local row r
// into the swizzled A tile, as dequant_w8 does.
__device__ __forceinline__ void widen_w16(const uint8_t* src, uint8_t* a_rows, int r, int half) {
  const int4 q0 = *reinterpret_cast<const int4*>(src);
  const int4 q1 = *reinterpret_cast<const int4*>(src + 16);
  const uint32_t words[8] = {static_cast<uint32_t>(q0.x), static_cast<uint32_t>(q0.y), static_cast<uint32_t>(q0.z),
                             static_cast<uint32_t>(q0.w), static_cast<uint32_t>(q1.x), static_cast<uint32_t>(q1.y),
                             static_cast<uint32_t>(q1.z), static_cast<uint32_t>(q1.w)};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t lo = words[2 * j], hi = words[2 * j + 1];
    const int c = 4 * half + j;
    *reinterpret_cast<float4*>(a_rows + r * 128 + ((c ^ (r & 7)) << 4)) =
        make_float4(__uint_as_float(lo << 16), __uint_as_float(lo & 0xffff0000u), __uint_as_float(hi << 16),
                    __uint_as_float(hi & 0xffff0000u));
  }
}

template <int BN, WeightFormat F>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tf32_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x,
                 float* __restrict__ out, const float* __restrict__ scales, int T, int N, int K, int group_size) {
  constexpr int B_BYTES = BN * BK * 4;
  extern __shared__ uint8_t raw_smem[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* a_tiles = base;
  uint8_t* b_tiles = base + STAGES * A_BYTES;
  uint8_t* w8_tiles = b_tiles + STAGES * B_BYTES;  // int8 / bf16 only: the weight staging area
  constexpr int WS_BYTES = staging_bytes(F);
  constexpr bool W8 = F == WeightFormat::kInt8;
  uint64_t* bars = reinterpret_cast<uint64_t*>(w8_tiles + STAGES * WS_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int n0 = blockIdx.x * BM;  // first weight row (output feature) of this CTA
  const int t0 = blockIdx.y * BN;  // first token
  const int kblocks = (K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_addr(&full[s]), 1);
      mbar_init(smem_addr(&empty[s]), 2);  // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    if (t == 0) {  // ---- TMA producer ----
      for (int kb = 0; kb < kblocks; ++kb) {
        const int s = kb % STAGES;
        const uint32_t ph = (kb / STAGES) & 1;
        mbar_wait(smem_addr(&empty[s]), ph ^ 1u);
        const uint32_t bar = smem_addr(&full[s]);
        // out-of-range rows / columns are zero-filled and still counted
        mbar_expect_tx(bar, (WS_BYTES ? WS_BYTES : A_BYTES) + B_BYTES);
        tma_load_2d(smem_addr(WS_BYTES ? w8_tiles + s * WS_BYTES : a_tiles + s * A_BYTES), &map_w, bar, kb * BK, n0);
        tma_load_2d(smem_addr(b_tiles + s * B_BYTES), &map_x, bar, kb * BK, t0);
      }
    }
    return;
  }
  // ---- consumers: warpgroup wg owns weight rows n0 + 64 (wg - 1) .. + 63 ----
  float d[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  const uint32_t a_off = static_cast<uint32_t>(wg - 1) * 64 * BK * 4;  // 8 KB: a multiple of the 1024-byte atom
  // W8: thread t dequantises 16 weights of local row t / 2; the row's scale for K block kb is one float
  const int dq_row = t >> 1, dq_half = t & 1;
  const int w_row = n0 + (wg - 1) * 64 + dq_row;
  const float* srow = (W8 && w_row < N) ? scales + static_cast<size_t>(w_row) * (K / group_size) : nullptr;
  auto scale_at = [&](int kb) { return srow != nullptr ? __ldg(srow + kb * BK / group_size) : 0.f; };
  float sc = W8 ? scale_at(0) : 0.f;
  for (int kb = 0; kb < kblocks; ++kb) {
    const int s = kb % STAGES;
    const float sc_next = (W8 && kb + 1 < kblocks) ? scale_at(kb + 1) : 0.f;
    mbar_wait(smem_addr(&full[s]), (kb / STAGES) & 1);
    // The tensor core truncates fp32 operands to tf32; round them to the nearest tf32 in place first, which halves
    // the per-operand error.  Each warpgroup rounds (or, for int8 weights, dequantises) its own 64 weight rows and
    // half of the token rows, which both read, so the two meet at a named barrier before the wgmma (async proxy)
    // reads the tiles.
    if constexpr (W8)
      dequant_w8(w8_tiles + s * WS_BYTES + ((wg - 1) * 64 + dq_row) * BK + dq_half * 16, a_tiles + s * A_BYTES + a_off,
                 dq_row, dq_half, sc);
    else if constexpr (F == WeightFormat::kBf16)
      widen_w16(w8_tiles + s * WS_BYTES + ((wg - 1) * 64 + dq_row) * BK * 2 + dq_half * 32,
                a_tiles + s * A_BYTES + a_off, dq_row, dq_half);
    else
      round_tf32(reinterpret_cast<float4*>(a_tiles + s * A_BYTES + a_off), 64 * BK / 4, t);
    round_tf32(reinterpret_cast<float4*>(b_tiles + s * B_BYTES + (wg - 1) * (B_BYTES / 2)), BN * BK / 8, t);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("bar.sync 1, 256;" ::: "memory");
    const uint64_t adesc = wgmma_desc_sw128(smem_addr(a_tiles + s * A_BYTES) + a_off);
    const uint64_t bdesc = wgmma_desc_sw128(smem_addr(b_tiles + s * B_BYTES));
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int k = 0; k < BK / WG_K; ++k)  // 32 bytes of K per instruction (2 descriptor units): inside the swizzle atom
      wgmma_tf32<BN>(d, adesc + 2 * k, bdesc + 2 * k, 1u);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    // the group of stage kb - 1 has retired: its tiles may be refilled
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
    if (kb > 0 && t == 0) mbar_arrive(smem_addr(&empty[(kb - 1) % STAGES]));
    sc = sc_next;
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");

  const int row = n0 + (wg - 1) * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int col = t0 + 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int r = row + 8 * (h >> 1), c = col + 8 * j + (h & 1);
      if (r < N && c < T) out[static_cast<size_t>(c) * N + r] = d[4 * j + h];
    }
  }
}

// cuTensorMapEncodeTiled comes from the driver (libcuda); it is looked up at run time so that the
// library links and loads on a machine without a driver (the build box).
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}
// 2-D tensor [rows, cols] (row-major, cols contiguous) of fp32 (elem 4, 128-byte swizzle), or of int8 or bf16
// (elem 1 or 2, no swizzle: the consumers read it back row by row), box [box_rows x 32 columns]
static int make_map(CUtensorMap* map, const void* ptr, int elem, int rows, int cols, int box_rows) {
  EncodeTiledFn fn = encode_tiled();
  if (fn == nullptr) return KLLM_E_NODEVICE;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * elem};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType type = elem == 1   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                   : elem == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16
                                               : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const CUresult r = fn(map, type, 2,
                        const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        elem != 4 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : KLLM_E_INVALID;
}

template <int BN, WeightFormat F>
static int launch(const float* x, const void* w, const float* scales, float* out, int T, int K, int N, int group_size,
                  cudaStream_t stream) {
  CUtensorMap map_w, map_x;
  if (int rc = make_map(&map_w, w, weight_bytes(F), N, K, BM)) return rc;
  if (int rc = make_map(&map_x, x, 4, T, K, BN)) return rc;
  const size_t smem = 1024 + static_cast<size_t>(STAGES) * (A_BYTES + BN * BK * 4 + staging_bytes(F)) + 128;
  static bool configured = false;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(gemm_tf32_kernel<BN, F>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  const dim3 grid((N + BM - 1) / BM, (T + BN - 1) / BN);
  gemm_tf32_kernel<BN, F><<<grid, THREADS, smem, stream>>>(map_w, map_x, out, scales, T, N, K, group_size);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

// token-block width: the smallest wgmma N that covers the tokens, 256 at most
template <WeightFormat F>
static int dispatch(const float* x, const void* w, const float* scales, float* out, int T, int K, int N, int group_size,
                    cudaStream_t s) {
  if (T <= 32) return launch<32, F>(x, w, scales, out, T, K, N, group_size, s);
  if (T <= 64) return launch<64, F>(x, w, scales, out, T, K, N, group_size, s);
  if (T <= 128) return launch<128, F>(x, w, scales, out, T, K, N, group_size, s);
  return launch<256, F>(x, w, scales, out, T, K, N, group_size, s);
}

}  // namespace tc
}  // namespace kllm

extern "C" int kllm_gemm_tf32(const float* x, const float* w, float* out, int n_tokens, int in_dim, int out_dim,
                              void* stream) {
  if (!x || !w || !out || n_tokens <= 0 || in_dim <= 0 || out_dim <= 0) return KLLM_E_INVALID;
  // TMA needs 16-byte aligned bases and row pitches
  if ((in_dim & 3) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15)) return KLLM_E_UNSUPPORTED;
  return kllm::tc::dispatch<kllm::WeightFormat::kF32>(x, w, nullptr, out, n_tokens, in_dim, out_dim, 0,
                                                     static_cast<cudaStream_t>(stream));
}

extern "C" int kllm_gemm_w8_tf32(const float* x, const int8_t* w, const float* scales, float* out, int n_tokens,
                                 int in_dim, int out_dim, int group_size, void* stream) {
  if (!x || !w || !scales || !out || n_tokens <= 0 || in_dim <= 0 || out_dim <= 0 || group_size <= 0)
    return KLLM_E_INVALID;
  // TMA needs 16-byte aligned bases and row pitches (in_dim bytes for the int8 rows); one scale per row and
  // 32-column K block needs whole groups per row and whole K blocks per group
  if ((in_dim % 16) || (in_dim % group_size) || (group_size % 32) || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(w) & 15))
    return KLLM_E_UNSUPPORTED;
  return kllm::tc::dispatch<kllm::WeightFormat::kInt8>(x, w, scales, out, n_tokens, in_dim, out_dim, group_size,
                                                      static_cast<cudaStream_t>(stream));
}

extern "C" int kllm_gemm_bf16_tf32(const float* x, const uint16_t* w, float* out, int n_tokens, int in_dim, int out_dim,
                                   void* stream) {
  if (!x || !w || !out || n_tokens <= 0 || in_dim <= 0 || out_dim <= 0) return KLLM_E_INVALID;
  // TMA needs 16-byte aligned bases and row pitches (2 in_dim bytes for the bf16 rows)
  if ((in_dim & 7) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15))
    return KLLM_E_UNSUPPORTED;
  return kllm::tc::dispatch<kllm::WeightFormat::kBf16>(x, w, nullptr, out, n_tokens, in_dim, out_dim, 0,
                                                      static_cast<cudaStream_t>(stream));
}
