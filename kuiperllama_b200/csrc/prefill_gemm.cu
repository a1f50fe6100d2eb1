// Batched GEMM for prompt prefill on the Hopper tensor cores (sm_90a):
//     out[T, N] = x[T, K] . w[N, K]^T        fp32 storage, TF32 multiply, fp32 accumulate in registers
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

template <int BN>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tf32_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_x,
                 float* __restrict__ out, int T, int N, int K) {
  constexpr int B_BYTES = BN * BK * 4;
  extern __shared__ uint8_t raw_smem[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* a_tiles = base;
  uint8_t* b_tiles = base + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_tiles + STAGES * B_BYTES);
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
        mbar_expect_tx(bar, A_BYTES + B_BYTES);  // out-of-range rows / columns are zero-filled and still counted
        tma_load_2d(smem_addr(a_tiles + s * A_BYTES), &map_w, bar, kb * BK, n0);
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
  for (int kb = 0; kb < kblocks; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(smem_addr(&full[s]), (kb / STAGES) & 1);
    // The tensor core truncates fp32 operands to tf32; round them to the nearest tf32 in place first, which halves
    // the per-operand error.  Each warpgroup rounds its own 64 weight rows and half of the token rows, which
    // both read, so the two meet at a named barrier before the wgmma (async proxy) reads the tiles.
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
// 2-D fp32 tensor [rows, cols] (row-major, cols contiguous), box [box_rows x 32 columns], 128-byte swizzle
static int make_map(CUtensorMap* map, const float* ptr, int rows, int cols, int box_rows) {
  EncodeTiledFn fn = encode_tiled();
  if (fn == nullptr) return KLLM_E_NODEVICE;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(cols) * 4};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : KLLM_E_INVALID;
}

template <int BN>
static int launch(const float* x, const float* w, float* out, int T, int K, int N, cudaStream_t stream) {
  CUtensorMap map_w, map_x;
  if (int rc = make_map(&map_w, w, N, K, BM)) return rc;
  if (int rc = make_map(&map_x, x, T, K, BN)) return rc;
  const size_t smem = 1024 + static_cast<size_t>(STAGES) * (A_BYTES + BN * BK * 4) + 128;
  static bool configured = false;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(gemm_tf32_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    configured = true;
  }
  const dim3 grid((N + BM - 1) / BM, (T + BN - 1) / BN);
  gemm_tf32_kernel<BN><<<grid, THREADS, smem, stream>>>(map_w, map_x, out, T, N, K);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

}  // namespace tc
}  // namespace kllm

extern "C" int kllm_gemm_tf32(const float* x, const float* w, float* out, int n_tokens, int in_dim, int out_dim,
                              void* stream) {
  if (!x || !w || !out || n_tokens <= 0 || in_dim <= 0 || out_dim <= 0) return KLLM_E_INVALID;
  // TMA needs 16-byte aligned bases and row pitches
  if ((in_dim & 3) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15)) return KLLM_E_UNSUPPORTED;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  using namespace kllm::tc;
  if (n_tokens <= 32) return launch<32>(x, w, out, n_tokens, in_dim, out_dim, s);
  if (n_tokens <= 64) return launch<64>(x, w, out, n_tokens, in_dim, out_dim, s);
  if (n_tokens <= 128) return launch<128>(x, w, out, n_tokens, in_dim, out_dim, s);
  return launch<256>(x, w, out, n_tokens, in_dim, out_dim, s);
}
