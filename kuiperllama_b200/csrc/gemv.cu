// Batch-1 weight-streaming GEMV for sm_90a, fp32 and int8-group weights, with the fused
// prologue/epilogues the decode loop needs (RMSNorm on the input; bias; residual add;
// SiLU*gate).  Replaces matmul_kernel_cu / matmul_kernel_cu_qint8
// (kuiper/source/op/kernels/cuda/matmul_kernel.cu:6-134) plus the rmsnorm / add / swiglu
// launches around them (llama3.cpp:600-720).
//
// Mapping.  The reference gives every output row a 128-thread CTA; lane t accumulates packs
// t, t+128, ... and a cub block reduction folds the 128 partials.  Here ONE WARP owns a row
// and each lane carries the partial sums of four of those 128 "virtual threads", so the
// floating-point result is bit-identical while a warp streams 2 KiB of contiguous weights per
// step with 128-bit loads and several rows in flight.  HBM-bound: 4 B (fp32) or 1.0625 B
// (int8 + scales) per multiply-add; tensor cores are deliberately not used (batch 1,
// 0.5 flop/B, and tf32/bf16 would break the 1e-4 / identical-token contract).
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>

#include "../../include/kllm_b200.h"
#include "kllm_device.cuh"
#include "kllm_host.h"

namespace kllm {

struct SegDev {
  const void* w;
  const float* scales;
  const float* bias;
  float* out;
  long long pos_stride;  // out += pos * pos_stride (KV-cache row of the current position)
  int rows;
};

struct GemvParams {
  const float* x;
  const float* norm_w;
  float* norm_out;
  const float* residual;
  float norm_eps;
  int in_dim;
  int group_size;
  int group_shift;  // log2(group_size) or -1
  int vec_ok;       // fp32: every weight row is 16-byte aligned (in_dim % 4 == 0, aligned bases)
  int n_seg;
  int units;  // output rows (or w1/w3 row pairs when swiglu)
  PosArg pos;
  SegDev seg[3];
};

constexpr int kGemvWarps = 8;
constexpr int kGemvThreads = kGemvWarps * 32;

// rmsnorm_kernel.cu:4-50 on the CTA's private copy of x in shared memory.  Executed by warp 0
// with the 128 virtual threads of the reference laid out as lane + 32*j.
__device__ __forceinline__ float rms_scale_ref(const float* xs, int n, float eps, int lane) {
  const int pack_num = n >> 2;
  const float4* xs4 = reinterpret_cast<const float4*>(xs);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int base = 0; base < pack_num; base += 128) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int idx = base + 32 * j + lane;
      if (idx < pack_num) {
        const float4 v = xs4[idx];
        float s = acc[j];
        s = __fmaf_rn(v.x, v.x, s);
        s = __fmaf_rn(v.y, v.y, s);
        s = __fmaf_rn(v.z, v.z, s);
        s = __fmaf_rn(v.w, v.w, s);
        acc[j] = s;
      }
    }
  }
  // scalar tail (n % 4), virtual thread t handles pack_off + t (+128k): only j = 0 can hit.
  for (int i = (pack_num << 2) + lane; i < n; i += 128) acc[0] = __fmaf_rn(xs[i], xs[i], acc[0]);
  float sum = block128_sum_vt(acc);
  sum = __shfl_sync(kFull, sum, 0);
  return rsqrtf(__fadd_rn(__fdiv_rn(sum, static_cast<float>(n)), eps));
}

template <int R, bool kInt8, bool kSwiglu>
__global__ void __launch_bounds__(kGemvThreads) gemv_kernel(const GemvParams p) {
  extern __shared__ __align__(16) float xs[];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int M = p.in_dim;

  // ---- stage x (optionally RMS-normalised) in shared memory --------------------------
  for (int i = threadIdx.x; i < M; i += kGemvThreads) xs[i] = p.x[i];
  __syncthreads();
  if (p.norm_w != nullptr) {
    __shared__ float s_scale;
    if (warp == 0) {
      const float sc = rms_scale_ref(xs, M, p.norm_eps, lane);
      if (lane == 0) s_scale = sc;
    }
    __syncthreads();
    const float sc = s_scale;
    const int pack_off = (M >> 2) << 2;
    for (int i = threadIdx.x; i < M; i += kGemvThreads) {
      // rmsnorm_kernel.cu:41-49: (scale*x)*w for packed elements, (w*x)*scale for the tail.
      const float v = (i < pack_off) ? __fmul_rn(__fmul_rn(sc, xs[i]), p.norm_w[i])
                                     : __fmul_rn(__fmul_rn(p.norm_w[i], xs[i]), sc);
      xs[i] = v;
      if (p.norm_out != nullptr && blockIdx.x == 0) p.norm_out[i] = v;
    }
    __syncthreads();
  }

  const int pack_num = M >> 2;
  const float4* xs4 = reinterpret_cast<const float4*>(xs);
  const long long pos = p.pos.get();
  constexpr int kRowsPerUnit = kSwiglu ? 2 : 1;
  constexpr int kUnits = R / kRowsPerUnit;
  const int warps_total = gridDim.x * kGemvWarps;
  const int gw = blockIdx.x * kGemvWarps + warp;

  for (int u0 = gw * kUnits; u0 < p.units; u0 += warps_total * kUnits) {
    // ---- resolve the R rows this warp owns ------------------------------------------
    const void* wrow[R];
    const float* srow[R];  // int8: scales base of the tensor
    long long ebase[R];    // int8: element index of the row start (for group lookup)
    bool live[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int u = u0 + r / kRowsPerUnit;
      live[r] = u < p.units;
      int seg = 0, row = live[r] ? u : 0;
      if (kSwiglu) {
        seg = r % 2;
      } else {
        if (p.n_seg > 1 && row >= p.seg[0].rows) {
          row -= p.seg[0].rows;
          seg = 1;
          if (p.n_seg > 2 && row >= p.seg[1].rows) {
            row -= p.seg[1].rows;
            seg = 2;
          }
        }
      }
      const long long e = static_cast<long long>(row) * M;
      ebase[r] = e;
      srow[r] = p.seg[seg].scales;
      wrow[r] = kInt8 ? static_cast<const void*>(static_cast<const int8_t*>(p.seg[seg].w) + e)
                      : static_cast<const void*>(static_cast<const float*>(p.seg[seg].w) + e);
    }

    float acc[R][4];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;

    if constexpr (!kInt8) {
      // virtual thread (lane + 32 j) <- packs base + 32 j + lane, base += 128
      const int full = p.vec_ok ? (pack_num & ~127) : 0;
      for (int base = 0; base < full; base += 128) {
        float4 wv[R][4];
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            wv[r][j] = ldg_stream_f4(static_cast<const float4*>(wrow[r]) + base + 32 * j + lane);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 xv = xs4[base + 32 * j + lane];
#pragma unroll
          for (int r = 0; r < R; ++r) acc[r][j] = __fadd_rn(dot4_ref(xv, wv[r][j]), acc[r][j]);
        }
      }
      // remainder packs (and every pack when rows are not 16-byte aligned: ragged in_dim --
      // the reference's float4 loads would fault there; same arithmetic, scalar loads)
      for (int base = full; base < pack_num; base += 128) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int idx = base + 32 * j + lane;
          if (idx < pack_num) {
            const float4 xv = xs4[idx];
#pragma unroll
            for (int r = 0; r < R; ++r) {
              float4 wv;
              if (p.vec_ok) {
                wv = ldg_stream_f4(static_cast<const float4*>(wrow[r]) + idx);
              } else {
                const float* wp = static_cast<const float*>(wrow[r]) + 4 * idx;
                wv = make_float4(__ldg(wp), __ldg(wp + 1), __ldg(wp + 2), __ldg(wp + 3));
              }
              acc[r][j] = __fadd_rn(dot4_ref(xv, wv), acc[r][j]);
            }
          }
        }
      }
      // scalar tail, matmul_kernel.cu:36-38 (FFMA into the lane's running sum)
      for (int i = (pack_num << 2) + lane; i < M; i += 128) {
#pragma unroll
        for (int r = 0; r < R; ++r)
          acc[r][0] = __fmaf_rn(xs[i], static_cast<const float*>(wrow[r])[i], acc[r][0]);
      }
    } else {
      // int8: virtual thread (4 lane + e) <- elements 128 k + 4 lane + e.
      // matmul_kernel.cu:70-74 as compiled: sdata = fma(x*scale, float(w), sdata).
      const int chunks = (M + 127) >> 7;
      for (int k = 0; k < chunks; ++k) {
        const int i = (k << 7) + (lane << 2);
        if (i < M) {
          const float4 xv = xs4[i >> 2];
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const uint32_t packed =
                ldg_stream_u32(reinterpret_cast<const uint32_t*>(static_cast<const int8_t*>(wrow[r]) + i));
            const long long e = ebase[r] + i;
            const long long g = p.group_shift >= 0 ? (e >> p.group_shift) : (e / p.group_size);
            const float sc = __ldg(srow[r] + g);
            float wf[4];
            int8x4_to_float(packed, wf);
            acc[r][0] = __fmaf_rn(__fmul_rn(xv.x, sc), wf[0], acc[r][0]);
            acc[r][1] = __fmaf_rn(__fmul_rn(xv.y, sc), wf[1], acc[r][1]);
            acc[r][2] = __fmaf_rn(__fmul_rn(xv.z, sc), wf[2], acc[r][2]);
            acc[r][3] = __fmaf_rn(__fmul_rn(xv.w, sc), wf[3], acc[r][3]);
          }
        }
      }
    }

    // ---- reduce + epilogue ------------------------------------------------------------
    float dot[R];
#pragma unroll
    for (int r = 0; r < R; ++r) dot[r] = kInt8 ? block128_sum_quad(acc[r]) : block128_sum_vt(acc[r]);

    if (lane == 0) {
#pragma unroll
      for (int un = 0; un < kUnits; ++un) {
        const int u = u0 + un;
        if (u >= p.units) break;
        if constexpr (kSwiglu) {
          // w1 row u and w3 row u -> swiglu_kernel.cu:16-21
          p.seg[0].out[u] = swiglu_ref(dot[2 * un], dot[2 * un + 1]);
        } else {
          int seg = 0, row = u;
          if (p.n_seg > 1 && row >= p.seg[0].rows) {
            row -= p.seg[0].rows;
            seg = 1;
            if (p.n_seg > 2 && row >= p.seg[1].rows) {
              row -= p.seg[1].rows;
              seg = 2;
            }
          }
          float v = dot[un];
          // matmul.cpp:74-77: add_kernel(out, bias) -> out + bias
          if (p.seg[seg].bias != nullptr) v = __fadd_rn(v, p.seg[seg].bias[row]);
          // llama3.cpp:683-684,719: add_kernel(x, matmul_out) -> x + matmul_out
          if (p.residual != nullptr) v = __fadd_rn(p.residual[row], v);
          p.seg[seg].out[pos * p.seg[seg].pos_stride + row] = v;
        }
      }
    }
  }
}

static int g_sm_count = 0;

static int sm_count() {
  if (g_sm_count == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      g_sm_count = 132;
  }
  return g_sm_count;
}

template <int R, bool kInt8, bool kSwiglu>
static int launch_gemv(const GemvParams& p, cudaStream_t stream) {
  constexpr int kUnits = R / (kSwiglu ? 2 : 1);
  const size_t smem = static_cast<size_t>(p.in_dim) * sizeof(float);
  auto kern = gemv_kernel<R, kInt8, kSwiglu>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  const int warps_needed = (p.units + kUnits - 1) / kUnits;
  int ctas = (warps_needed + kGemvWarps - 1) / kGemvWarps;
  // persistent-ish: at most 4 CTAs (32 warps) per SM, grid a multiple of the SM count
  const int cap = sm_count() * 4;
  if (ctas > cap) ctas = cap;
  if (ctas < 1) ctas = 1;
  kern<<<ctas, kGemvThreads, smem, stream>>>(p);
  count_launch();
  return static_cast<int>(cudaGetLastError());
}

int gemv_dispatch(const kllm_gemv_job* job, const GemvExtra& extra, cudaStream_t stream) {
  if (job == nullptr || job->x == nullptr || job->in_dim <= 0) return KLLM_E_INVALID;
  if (job->n_seg < 1 || job->n_seg > 3) return KLLM_E_INVALID;
  const bool int8 = job->group_size > 0;
  if (job->swiglu_pair && (job->n_seg != 2 || job->seg[0].rows != job->seg[1].rows ||
                           job->residual != nullptr))
    return KLLM_E_INVALID;
  if (int8 && ((job->in_dim & 3) != 0 || (job->group_size & 3) != 0)) return KLLM_E_UNSUPPORTED;
  if (static_cast<size_t>(job->in_dim) * sizeof(float) > 200 * 1024) return KLLM_E_UNSUPPORTED;

  GemvParams p{};
  p.x = job->x;
  p.norm_w = job->norm_w;
  p.norm_out = job->norm_out;
  p.norm_eps = job->norm_eps;
  p.residual = job->residual;
  p.in_dim = job->in_dim;
  p.group_size = job->group_size;
  p.group_shift = -1;
  if (int8 && (job->group_size & (job->group_size - 1)) == 0) {
    int s = 0;
    while ((1 << s) < job->group_size) ++s;
    p.group_shift = s;
  }
  p.n_seg = job->n_seg;
  p.pos = extra.pos;
  p.vec_ok = (job->in_dim & 3) == 0;
  int total = 0;
  for (int s = 0; s < job->n_seg; ++s) {
    const kllm_gemv_seg& g = job->seg[s];
    if (g.w == nullptr || g.rows <= 0) return KLLM_E_INVALID;
    if (int8 && g.scales == nullptr) return KLLM_E_INVALID;
    if (g.out == nullptr && !(job->swiglu_pair && s == 1)) return KLLM_E_INVALID;
    if ((reinterpret_cast<uintptr_t>(g.w) & (int8 ? 3 : 15)) != 0) {
      if (int8) return KLLM_E_UNSUPPORTED;
      p.vec_ok = 0;
    }
    p.seg[s] = SegDev{g.w, g.scales, g.bias, g.out, extra.pos_stride[s], g.rows};
    total += g.rows;
  }
  p.units = job->swiglu_pair ? job->seg[0].rows : total;

  // Rows per warp: enough independent 128-bit loads in flight per lane (R*4) while still
  // giving every SM work for the small matrices (kv projections: 256 rows).
  const int warps_1wave = sm_count() * kGemvWarps;
  if (job->swiglu_pair) {
    if (int8) return p.units >= warps_1wave * 2 ? launch_gemv<4, true, true>(p, stream)
                                                : launch_gemv<2, true, true>(p, stream);
    return p.units >= warps_1wave * 2 ? launch_gemv<4, false, true>(p, stream)
                                      : launch_gemv<2, false, true>(p, stream);
  }
  if (int8) {
    if (p.units >= warps_1wave * 4) return launch_gemv<4, true, false>(p, stream);
    if (p.units >= warps_1wave * 2) return launch_gemv<2, true, false>(p, stream);
    return launch_gemv<1, true, false>(p, stream);
  }
  if (p.units >= warps_1wave * 4) return launch_gemv<4, false, false>(p, stream);
  if (p.units >= warps_1wave * 2) return launch_gemv<2, false, false>(p, stream);
  return launch_gemv<1, false, false>(p, stream);
}

}  // namespace kllm

extern "C" {

int kllm_gemv_fused(const kllm_gemv_job* job, void* stream) {
  return kllm::gemv_dispatch(job, kllm::GemvExtra{}, static_cast<cudaStream_t>(stream));
}

int kllm_gemv_f32(const float* x, const float* w, float* out, int in_dim, int out_dim,
                  void* stream) {
  if (!x || !w || !out || in_dim <= 0 || out_dim <= 0) return KLLM_E_INVALID;
  kllm_gemv_job job{};
  job.x = x;
  job.in_dim = in_dim;
  job.n_seg = 1;
  job.seg[0].w = w;
  job.seg[0].out = out;
  job.seg[0].rows = out_dim;
  return kllm_gemv_fused(&job, stream);
}

int kllm_gemv_w8(const float* x, const int8_t* w, const float* scales, float* out, int in_dim,
                 int out_dim, int group_size, void* stream) {
  if (!x || !w || !scales || !out || in_dim <= 0 || out_dim <= 0 || group_size <= 0)
    return KLLM_E_INVALID;
  kllm_gemv_job job{};
  job.x = x;
  job.in_dim = in_dim;
  job.group_size = group_size;
  job.n_seg = 1;
  job.seg[0].w = w;
  job.seg[0].scales = scales;
  job.seg[0].out = out;
  job.seg[0].rows = out_dim;
  return kllm_gemv_fused(&job, stream);
}

}  // extern "C"
