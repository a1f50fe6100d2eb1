/* kuiper_oracle.c -- CPU restatement of the KuiperLLama decode hot path (see kuiper_oracle.h).
 *
 * TEST INFRASTRUCTURE ONLY: never linked into, loaded by, or called from the product library.
 * Citations are relative to the reference checkout's root.
 */
#define _GNU_SOURCE
#include "kuiper_oracle.h"

#include <dlfcn.h>
#include <fcntl.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------------------------- */
/* matmul                                                                                */
/* ------------------------------------------------------------------------------------- */
static int g_matmul_mode = KO_MATMUL_STRICT;
typedef void (*cblas_sgemv_fn)(int order, int trans, int m, int n, float alpha, const float* a,
                               int lda, const float* x, int incx, float beta, float* y, int incy);
static cblas_sgemv_fn g_sgemv = NULL;
static void* g_blas_handle = NULL;

void ko_set_matmul_mode(int mode) { g_matmul_mode = mode; }

int ko_set_blas_library(const char* so) {
  void* h = dlopen(so, RTLD_NOW | RTLD_LOCAL);
  if (!h) return -1;
  void* f = dlsym(h, "cblas_sgemv");
  if (!f) f = dlsym(h, "scipy_cblas_sgemv");
  if (!f) return -2;
  g_sgemv = (cblas_sgemv_fn)f;
  g_blas_handle = h;
  return 0;
}

/* Thread count of the TIMED baseline, set through the libraries' own APIs so that an inherited
 * OMP_NUM_THREADS=1 (torchrun exports it) cannot silently serialise the reference arm.  Returns
 * what the BLAS reports afterwards (0: no BLAS loaded). */
int ko_set_num_threads(int n) {
  if (n < 1) n = 1;
#ifdef _OPENMP
  omp_set_num_threads(n);
#endif
  if (!g_blas_handle) return 0;
  typedef void (*set_fn)(int);
  typedef int (*get_fn)(void);
  set_fn set = (set_fn)dlsym(g_blas_handle, "openblas_set_num_threads");
  if (!set) set = (set_fn)dlsym(g_blas_handle, "scipy_openblas_set_num_threads");
  if (set) set(n);
  get_fn get = (get_fn)dlsym(g_blas_handle, "openblas_get_num_threads");
  if (!get) get = (get_fn)dlsym(g_blas_handle, "scipy_openblas_get_num_threads");
  return get ? get() : 0;
}

int ko_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* cpu/matmul_kernel.cpp:37-40: weight_mat is the row-major [K(out), M(in)] block viewed as a
 * column-major M x K arma::fmat; output = (x^T W^T) * scale, i.e. one dot product per row. */
void ko_matmul_f32(const float* x, const float* w, float* out, int M, int K, float scale) {
  if (g_matmul_mode == KO_MATMUL_FAST) {
    if (g_sgemv && K >= 64) {
      /* CblasRowMajor=101, CblasNoTrans=111: y = alpha*A*x, A is K x M row-major. */
      g_sgemv(101, 111, K, M, scale, w, M, x, 1, 0.f, out, 1);
      return;
    }
#pragma omp parallel for schedule(static) if (K >= 64)
    for (int p = 0; p < K; ++p) {
      const float* row = w + (size_t)p * M;
      float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      int i = 0;
      for (; i + 8 <= M; i += 8)
        for (int j = 0; j < 8; ++j) acc[j] += row[i + j] * x[i + j];
      float s = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
      for (; i < M; ++i) s += row[i] * x[i];
      out[p] = s * scale;
    }
    return;
  }
  for (int p = 0; p < K; ++p) {
    const float* row = w + (size_t)p * M;
    float s = 0.f;
    for (int i = 0; i < M; ++i) s += x[i] * row[i];
    out[p] = s * scale;
  }
}

/* cuda/matmul_kernel.cu:68-74.  The reference has no CPU int8 matmul
 * (kernels_interfaces.cpp:54-61); this restates the per-element arithmetic
 * x[i] * scales[group] * (float)w in that association, summed left to right. */
void ko_matmul_w8(const float* x, const int8_t* w, const float* scales, float* out, int M, int K,
                  int group_size) {
#pragma omp parallel for schedule(static) if (g_matmul_mode == KO_MATMUL_FAST && K >= 64)
  for (int p = 0; p < K; ++p) {
    float s = 0.f;
    for (int i = 0; i < M; ++i) {
      const int64_t idx = (int64_t)p * M + i;
      s += x[i] * scales[idx / group_size] * (float)w[idx];
    }
    out[p] = s;
  }
}

/* cub::BlockReduce<float,128>::Sum with the default BLOCK_REDUCE_WARP_REDUCTIONS algorithm
 * (CCCL shipped with CUDA 12.9): each warp runs a shuffle-down tree with offsets 1,2,4,8,16
 * (lane i += lane i+offset while i+offset < 32), then thread 0 adds the warp aggregates
 * sequentially: ((w0 + w1) + w2) + w3.  Verified bit-for-bit on the GPU against
 * oracle/_ref (tests/test_kernels_gpu.py::test_cuda_order_model). */
static float cub_block_sum_128(float v[128]) {
  float agg[4];
  for (int w = 0; w < 4; ++w) {
    float* l = v + 32 * w;
    for (int off = 1; off < 32; off <<= 1) {
      float nxt[32];
      for (int i = 0; i < 32; ++i) nxt[i] = (i + off < 32) ? l[i] + l[i + off] : l[i];
      memcpy(l, nxt, sizeof(nxt));
    }
    agg[w] = l[0];
  }
  return ((agg[0] + agg[1]) + agg[2]) + agg[3];
}

/* cuda/matmul_kernel.cu:27-38: lane t walks float4 packs t, t+128, ...; each pack contributes
 * part = x.x*w.x + x.y*w.y + x.z*w.z + x.w*w.w, which nvcc 12.9 (-fmad=true default) contracts
 * for sm_90a to fma(x.w,w.w, fma(x.z,w.z, fma(x.x,w.x, x.y*w.y))) -- read off the SASS of
 * oracle/_ref (FMUL y; FFMA x; FFMA z; FFMA w; FADD acc) -- then sdata[t] += part (plain add). */
void ko_matmul_f32_cuda_order(const float* x, const float* w, float* out, int M, int K) {
  const int pack_num = M / 4, pack_off = pack_num * 4;
  for (int p = 0; p < K; ++p) {
    const float* row = w + (size_t)p * M;
    float lane[128];
    for (int t = 0; t < 128; ++t) {
      float s = 0.f;
      for (int i = t; i < pack_num; i += 128) {
        const float* a = x + 4 * i;
        const float* b = row + 4 * i;
        float part = a[1] * b[1];
        part = fmaf(a[0], b[0], part);
        part = fmaf(a[2], b[2], part);
        part = fmaf(a[3], b[3], part);
        s += part;
      }
      for (int i = pack_off + t; i < M; i += 128) s = fmaf(x[i], row[i], s);
      lane[t] = s;
    }
    out[p] = cub_block_sum_128(lane);
  }
}

/* cuda/matmul_kernel.cu:68-74 in device order: lane t walks i = t, t+128, ...;
 * sdata[t] += (x[i]*scale)*float(w) -> contracted to fma(x*scale, float(w), sdata). */
void ko_matmul_w8_cuda_order(const float* x, const int8_t* w, const float* scales, float* out,
                             int M, int K, int group_size) {
  for (int p = 0; p < K; ++p) {
    float lane[128];
    for (int t = 0; t < 128; ++t) {
      float s = 0.f;
      for (int i = t; i < M; i += 128) {
        const int64_t idx = (int64_t)p * M + i;
        const float xs = x[i] * scales[idx / group_size];
        s = fmaf(xs, (float)w[idx], s);
      }
      lane[t] = s;
    }
    out[p] = cub_block_sum_128(lane);
  }
}

/* ------------------------------------------------------------------------------------- */
/* element-wise / small ops                                                              */
/* ------------------------------------------------------------------------------------- */
float ko_flavour_eps(int flavour) { return flavour == KO_FLAVOUR_QWEN2 ? 1e-6f : 1e-5f; }

float ko_flavour_theta(int flavour) {
  if (flavour == KO_FLAVOUR_LLAMA3) return 500000.0f;
  if (flavour == KO_FLAVOUR_QWEN2) return 1000000.0f;
  return 10000.0f;
}

/* cpu/rmsnorm_kernel.cpp:26-32: mean(x^2) + eps, 1/sqrt, w % (r * x). */
void ko_rmsnorm(const float* x, const float* w, float* out, int n, float eps) {
  float ss = 0.f;
  for (int i = 0; i < n; ++i) ss += x[i] * x[i];
  const float mean = ss / (float)n + eps;
  const float r = 1.f / sqrtf(mean);
  for (int i = 0; i < n; ++i) out[i] = w[i] * (r * x[i]);
}

/* cpu/add_kernel.cpp:18 */
void ko_add(const float* a, const float* b, float* out, int n) {
  for (int i = 0; i < n; ++i) out[i] = a[i] + b[i];
}

/* cpu/swiglu_kernel.cpp:21-22: x1 %= 1/(1+exp(-x1)); out = x1 % x3. */
void ko_swiglu(const float* x1, const float* x3, float* out, int n) {
  for (int i = 0; i < n; ++i) {
    const float g = x1[i] * (1.0f / (1.0f + expf(-x1[i])));
    out[i] = g * x3[i];
  }
}

/* cpu/softmax_kernel.cpp:4-15 */
void ko_softmax_inplace(float* x, int n) {
  float mx = x[0];
  for (int i = 1; i < n; ++i)
    if (x[i] > mx) mx = x[i];
  float sum = 0.f;
  for (int i = 0; i < n; ++i) {
    x[i] = expf(x[i] - mx);
    sum += x[i];
  }
  for (int i = 0; i < n; ++i) x[i] = x[i] / sum;
}

/* cpu/scale_sum_kernel.cpp:17-21: out += score[i] * value[i*stride .. +size), i = 0..pos. */
void ko_scale_sum(const float* value, const float* score, float* out, int pos, int size,
                  int stride) {
  for (int i = 0; i <= pos; ++i) {
    const float* v = value + (size_t)i * stride;
    for (int d = 0; d < size; ++d) out[d] += score[i] * v[d];
  }
}

/* cpu/emb_kernel.cpp:14-28 */
void ko_embedding(const int32_t* tokens, int n_tokens, const float* table, float* out, int dim,
                  int vocab) {
  for (int t = 0; t < n_tokens; ++t) {
    const int32_t tok = tokens[t];
    if (tok < 0 || tok >= vocab) continue; /* reference LOG(FATAL)s above vocab */
    memcpy(out + (size_t)t * dim, table + (size_t)tok * dim, sizeof(float) * dim);
  }
}

/* sampler/argmax_sampler.cpp:7: std::max_element -> first maximum. */
int64_t ko_argmax(const float* logits, int64_t n) {
  int64_t best = 0;
  for (int64_t i = 1; i < n; ++i)
    if (logits[i] > logits[best]) best = i;
  return best;
}

/* cpu/rope_kernel.cpp:4-17 / 44-57 / 84-97 (identical up to theta). */
void ko_sincos(int head_size, int seq_len, float theta, float* sin_cache, float* cos_cache) {
  for (int pos = 0; pos < seq_len; ++pos) {
    for (int d = 0; d < head_size; ++d) {
      const float freq = 1.0f / powf(theta, (float)d / (float)head_size);
      const float val = (float)pos * freq;
      sin_cache[pos * head_size + d] = sinf(val);
      cos_cache[pos * head_size + d] = cosf(val);
    }
  }
}

/* cpu/rope_kernel.cpp:99-121 (default, interleaved pairs) and :19-42 / :59-82 (half-split).
 * The half-split loops start at head_dim = i % head_size, which is always 0 since i steps by
 * head_size. */
void ko_rope(int flavour, int dim, int kv_dim, int head_size, float* q, float* k, int pos,
             const float* sin_cache, const float* cos_cache) {
  if (flavour == KO_FLAVOUR_LLAMA2) {
    for (int i = 0; i < dim; i += 2) {
      const int hd = i % head_size;
      const float fci = sin_cache[pos * head_size + hd];
      const float fcr = cos_cache[pos * head_size + hd];
      const int rotn = i < kv_dim ? 2 : 1;
      for (int v = 0; v < rotn; ++v) {
        float* vec = v == 0 ? q : k;
        const float v0 = vec[i], v1 = vec[i + 1];
        vec[i] = v0 * fcr - v1 * fci;
        vec[i + 1] = v0 * fci + v1 * fcr;
      }
    }
    return;
  }
  const int half = head_size / 2;
  for (int i = 0; i < dim; i += head_size) {
    for (int hd = 0; hd < half; ++hd) {
      const float fci = sin_cache[pos * head_size + hd * 2];
      const float fcr = cos_cache[pos * head_size + hd * 2];
      const int rotn = i < kv_dim ? 2 : 1;
      for (int v = 0; v < rotn; ++v) {
        float* vec = v == 0 ? q : k;
        const float v0 = vec[i + hd], v1 = vec[i + hd + half];
        vec[i + hd] = v0 * fcr - v1 * fci;
        vec[i + hd + half] = v0 * fci + v1 * fcr;
      }
    }
  }
}

/* cpu/mha_kernel.cpp:10-60: per head, score[t] = (q . k_t) * 1/sqrt(hs) via the matmul
 * kernel; softmax; out = 0; scale_sum over the value rows. */
void ko_mha(int pos, int head_num, int layer_index, int seq_len, int kv_dim, int kv_mul,
            int head_size, float* out, const float* q, float* score, const float* key_cache,
            const float* value_cache) {
  const size_t layer_offset = (size_t)layer_index * seq_len * kv_dim;
  const float scale = 1.f / sqrtf((float)head_size);
  const int saved_mode = g_matmul_mode;
  g_matmul_mode = KO_MATMUL_STRICT; /* head_size-long dots: always the plain loop */
  for (int h = 0; h < head_num; ++h) {
    float* score_head = score + (size_t)h * seq_len;
    const float* q_head = q + (size_t)h * head_size;
    const int head_off = (h / kv_mul) * head_size;
    for (int t = 0; t <= pos; ++t) {
      const float* key = key_cache + layer_offset + (size_t)t * kv_dim + head_off;
      ko_matmul_f32(q_head, key, score_head + t, head_size, 1, scale);
    }
    ko_softmax_inplace(score_head, pos + 1);
    float* out_head = out + (size_t)h * head_size;
    memset(out_head, 0, sizeof(float) * head_size);
    ko_scale_sum(value_cache + layer_offset + head_off, score_head, out_head, pos, head_size,
                 kv_dim);
  }
  g_matmul_mode = saved_mode;
}

/* tools/export.py:49-73 quantize_q80 (torch: w.abs().max per group / 127, round half-even
 * via torch.round, int8).  nearbyintf under the default rounding mode = round-half-even. */
void ko_quantize_q80(const float* w, int64_t n, int group_size, int8_t* q, float* scales) {
  const int64_t groups = n / group_size;
  for (int64_t g = 0; g < groups; ++g) {
    const float* src = w + g * group_size;
    float wmax = 0.f;
    for (int i = 0; i < group_size; ++i) {
      const float a = fabsf(src[i]);
      if (a > wmax) wmax = a;
    }
    const float scale = wmax / 127.0f;
    scales[g] = scale;
    for (int i = 0; i < group_size; ++i) {
      const float quant = src[i] / scale;
      q[g * group_size + i] = (int8_t)nearbyintf(quant);
    }
  }
}

/* ------------------------------------------------------------------------------------- */
/* whole model                                                                           */
/* ------------------------------------------------------------------------------------- */
typedef struct {
  const void* w;       /* fp32 or int8 weights */
  const float* scales; /* int8 only */
  const float* bias;   /* qwen qkv only */
} ko_linear;

struct ko_model {
  ko_config cfg;
  int fd;
  size_t file_size;
  void* map;
  const float* tok_emb;
  const float *attn_norm, *ffn_norm, *final_norm; /* [L,dim],[L,dim],[dim] */
  ko_linear *wq, *wk, *wv, *wo, *w1, *w2, *w3;     /* [L] each */
  ko_linear wcls;
  /* activations (llama3.cpp:425-500), aliasing kept explicit below */
  float *x, *rms_out, *query, *w1_out, *w3_out, *score, *logits;
  float *key_cache, *value_cache, *sin_cache, *cos_cache;
};

static void linear_forward(const ko_model* m, const ko_linear* l, const float* x, float* out,
                           int in_dim, int out_dim) {
  if (m->cfg.is_quant) {
    ko_matmul_w8(x, (const int8_t*)l->w, l->scales, out, in_dim, out_dim, m->cfg.group_size);
  } else {
    ko_matmul_f32(x, (const float*)l->w, out, in_dim, out_dim, 1.f);
  }
  if (l->bias) ko_add(out, l->bias, out, out_dim); /* matmul.cpp:74-77 */
}

const ko_config* ko_model_config(const ko_model* m) { return &m->cfg; }
const float* ko_model_key_cache(const ko_model* m) { return m->key_cache; }
const float* ko_model_value_cache(const ko_model* m) { return m->value_cache; }

ko_model* ko_model_open(const char* path, int is_quant, int flavour) {
  int fd = open(path, O_RDONLY);
  if (fd < 0) return NULL;
  struct stat st;
  if (fstat(fd, &st) != 0) {
    close(fd);
    return NULL;
  }
  void* map = mmap(NULL, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
  if (map == MAP_FAILED) {
    close(fd);
    return NULL;
  }
  ko_model* m = (ko_model*)calloc(1, sizeof(ko_model));
  m->fd = fd;
  m->file_size = (size_t)st.st_size;
  m->map = map;
  const int32_t* hdr = (const int32_t*)map; /* model.cpp:57-69 */
  ko_config* c = &m->cfg;
  c->dim = hdr[0];
  c->hidden_dim = hdr[1];
  c->layer_num = hdr[2];
  c->head_num = hdr[3];
  c->kv_head_num = hdr[4];
  c->seq_len = hdr[6];
  c->is_quant = is_quant;
  c->group_size = is_quant ? hdr[7] : 1;
  c->flavour = flavour;
  /* model.cpp:125-151 */
  c->kv_dim = (c->dim * c->kv_head_num) / c->head_num;
  c->kv_mul = c->head_num / c->kv_head_num;
  c->head_size = c->dim / c->head_num;
  c->shared_classifier = hdr[5] > 0;
  c->vocab_size = abs(hdr[5]);

  const int L = c->layer_num, dim = c->dim, kvd = c->kv_dim, hid = c->hidden_dim,
            V = c->vocab_size;
  m->wq = calloc(L, sizeof(ko_linear));
  m->wk = calloc(L, sizeof(ko_linear));
  m->wv = calloc(L, sizeof(ko_linear));
  m->wo = calloc(L, sizeof(ko_linear));
  m->w1 = calloc(L, sizeof(ko_linear));
  m->w2 = calloc(L, sizeof(ko_linear));
  m->w3 = calloc(L, sizeof(ko_linear));
  const int qkv_bias = (flavour == KO_FLAVOUR_QWEN2 || flavour == KO_FLAVOUR_QWEN2FILE) && !is_quant;

  if (!is_quant) {
    /* llama3.cpp:290-423 (fp32 v0); qwen2.cpp:304-333 interleaves a bias after each of
     * wq/wk/wv per layer. */
    const float* p = (const float*)((const char*)map + 7 * sizeof(int32_t));
    m->tok_emb = p;
    p += (size_t)V * dim;
    m->attn_norm = p;
    p += (size_t)L * dim;
    for (int l = 0; l < L; ++l) {
      m->wq[l].w = p;
      p += (size_t)dim * dim;
      if (qkv_bias) {
        m->wq[l].bias = p;
        p += dim;
      }
    }
    for (int l = 0; l < L; ++l) {
      m->wk[l].w = p;
      p += (size_t)kvd * dim;
      if (qkv_bias) {
        m->wk[l].bias = p;
        p += kvd;
      }
    }
    for (int l = 0; l < L; ++l) {
      m->wv[l].w = p;
      p += (size_t)kvd * dim;
      if (qkv_bias) {
        m->wv[l].bias = p;
        p += kvd;
      }
    }
    for (int l = 0; l < L; ++l) {
      m->wo[l].w = p;
      p += (size_t)dim * dim;
    }
    m->ffn_norm = p;
    p += (size_t)L * dim;
    for (int l = 0; l < L; ++l) {
      m->w1[l].w = p;
      p += (size_t)hid * dim;
    }
    for (int l = 0; l < L; ++l) {
      m->w2[l].w = p;
      p += (size_t)dim * hid;
    }
    for (int l = 0; l < L; ++l) {
      m->w3[l].w = p;
      p += (size_t)hid * dim;
    }
    m->final_norm = p;
    p += dim;
    p += (size_t)c->seq_len * c->head_size; /* freqs_cos + freqs_sin, llama3.cpp:367-368 */
    m->wcls.w = c->shared_classifier ? (const void*)m->tok_emb : (const void*)p;
  } else {
    /* llama3.cpp:184-288 (int8 v3): q block then fp32 scales per tensor per layer. */
    const int g = c->group_size;
    const char* p = (const char*)map + 8 * sizeof(int32_t);
#define KO_TAKE_Q(dst, rows, cols)                                   \
  do {                                                               \
    (dst).w = p;                                                     \
    p += (size_t)(rows) * (cols);                                    \
    (dst).scales = (const float*)p;                                  \
    p += ((size_t)(rows) * (cols) / g) * sizeof(float);              \
  } while (0)
    for (int l = 0; l < L; ++l) KO_TAKE_Q(m->wq[l], dim, dim);
    for (int l = 0; l < L; ++l) KO_TAKE_Q(m->wk[l], kvd, dim);
    for (int l = 0; l < L; ++l) KO_TAKE_Q(m->wv[l], kvd, dim);
    for (int l = 0; l < L; ++l) KO_TAKE_Q(m->wo[l], dim, dim);
    for (int l = 0; l < L; ++l) KO_TAKE_Q(m->w1[l], hid, dim);
    for (int l = 0; l < L; ++l) KO_TAKE_Q(m->w2[l], dim, hid);
    for (int l = 0; l < L; ++l) KO_TAKE_Q(m->w3[l], hid, dim);
    if (!c->shared_classifier) {
      KO_TAKE_Q(m->wcls, V, dim);
    } else {
      /* llama3.cpp:259-263: the reference points the int8 classifier at the fp32 embedding
       * (a known defect, SURVEY.md 8c); shared-classifier int8 files are rejected here. */
      fprintf(stderr, "ko_model_open: int8 + shared classifier is not supported\n");
      ko_model_close(m);
      return NULL;
    }
#undef KO_TAKE_Q
    const float* f = (const float*)p;
    m->tok_emb = f;
    f += (size_t)V * dim;
    m->attn_norm = f;
    f += (size_t)L * dim;
    m->ffn_norm = f;
    f += (size_t)L * dim;
    m->final_norm = f;
  }

  /* llama3.cpp:425-500 */
  m->x = calloc(dim, sizeof(float));
  m->rms_out = calloc(dim, sizeof(float));
  m->query = calloc(dim, sizeof(float));
  m->w1_out = calloc(hid, sizeof(float));
  m->w3_out = calloc(hid, sizeof(float));
  m->score = calloc((size_t)c->head_num * c->seq_len, sizeof(float));
  m->logits = calloc(V, sizeof(float));
  m->key_cache = calloc((size_t)L * c->seq_len * kvd, sizeof(float));
  m->value_cache = calloc((size_t)L * c->seq_len * kvd, sizeof(float));
  m->sin_cache = calloc((size_t)c->seq_len * c->head_size, sizeof(float));
  m->cos_cache = calloc((size_t)c->seq_len * c->head_size, sizeof(float));
  ko_sincos(c->head_size, c->seq_len, ko_flavour_theta(flavour), m->sin_cache, m->cos_cache);
  return m;
}

void ko_model_close(ko_model* m) {
  if (!m) return;
  free(m->wq), free(m->wk), free(m->wv), free(m->wo), free(m->w1), free(m->w2), free(m->w3);
  free(m->x), free(m->rms_out), free(m->query), free(m->w1_out), free(m->w3_out);
  free(m->score), free(m->logits), free(m->key_cache), free(m->value_cache);
  free(m->sin_cache), free(m->cos_cache);
  if (m->map) munmap(m->map, m->file_size);
  if (m->fd >= 0) close(m->fd);
  free(m);
}

const void* ko_model_tensor(const ko_model* m, const char* name, int layer,
                            const float** scales_out) {
  const ko_linear* l = NULL;
  const int dim = m->cfg.dim;
  if (scales_out) *scales_out = NULL;
  if (!strcmp(name, "tok_emb")) return m->tok_emb;
  if (!strcmp(name, "attn_norm")) return m->attn_norm + (size_t)layer * dim;
  if (!strcmp(name, "ffn_norm")) return m->ffn_norm + (size_t)layer * dim;
  if (!strcmp(name, "final_norm")) return m->final_norm;
  if (!strcmp(name, "wq")) l = &m->wq[layer];
  else if (!strcmp(name, "wk")) l = &m->wk[layer];
  else if (!strcmp(name, "wv")) l = &m->wv[layer];
  else if (!strcmp(name, "wo")) l = &m->wo[layer];
  else if (!strcmp(name, "w1")) l = &m->w1[layer];
  else if (!strcmp(name, "w2")) l = &m->w2[layer];
  else if (!strcmp(name, "w3")) l = &m->w3[layer];
  else if (!strcmp(name, "wcls")) l = &m->wcls;
  else if (!strcmp(name, "bq")) return m->wq[layer].bias;
  else if (!strcmp(name, "bk")) return m->wk[layer].bias;
  else if (!strcmp(name, "bv")) return m->wv[layer].bias;
  if (!l) return NULL;
  if (scales_out) *scales_out = l->scales;
  return l->w;
}

/* llama3.cpp:147-167 forward, :642-650 predict, :733-745 post_processing.
 * Buffer aliasing of llama3.cpp:456-489 is kept: kOutputRMSNorm == kOutputMHA == kW2Output ==
 * kFFNRMSNorm (rms_out), kAttnOutput == kQuery (query). */
int ko_model_step(ko_model* m, int token, int pos, float* logits_out) {
  const ko_config* c = &m->cfg;
  const int dim = c->dim, kvd = c->kv_dim, hid = c->hidden_dim, L = c->layer_num;
  const float eps = ko_flavour_eps(c->flavour);
  /* embedding + fill_input (llama3.cpp:578-598, model.cpp:245-263): x is the embedding row,
   * updated in place by the residual adds. */
  int32_t tok = token;
  ko_embedding(&tok, 1, m->tok_emb, m->x, dim, c->vocab_size);

  for (int l = 0; l < L; ++l) {
    /* attention_rms :600-609 */
    ko_rmsnorm(m->x, m->attn_norm + (size_t)l * dim, m->rms_out, dim, eps);
    /* attention_qkv :611-640 -- k, v written straight into the cache row (slice_kv_cache) */
    float* k = m->key_cache + ((size_t)l * c->seq_len + pos) * kvd;
    float* v = m->value_cache + ((size_t)l * c->seq_len + pos) * kvd;
    linear_forward(m, &m->wq[l], m->rms_out, m->query, dim, dim);
    linear_forward(m, &m->wk[l], m->rms_out, k, dim, kvd);
    linear_forward(m, &m->wv[l], m->rms_out, v, dim, kvd);
    ko_rope(c->flavour == KO_FLAVOUR_QWEN2FILE ? KO_FLAVOUR_LLAMA2 : c->flavour, dim, kvd,
            c->head_size, m->query, k, pos, m->sin_cache, m->cos_cache);
    /* attention_mha :652-676 */
    ko_mha(pos, c->head_num, l, c->seq_len, kvd, c->kv_mul, c->head_size, m->rms_out, m->query,
           m->score, m->key_cache, m->value_cache);
    linear_forward(m, &m->wo[l], m->rms_out, m->query, dim, dim);
    /* feed_forward :678-720 */
    ko_add(m->x, m->query, m->x, dim);
    ko_rmsnorm(m->x, m->ffn_norm + (size_t)l * dim, m->rms_out, dim, eps);
    linear_forward(m, &m->w1[l], m->rms_out, m->w1_out, dim, hid);
    linear_forward(m, &m->w3[l], m->rms_out, m->w3_out, dim, hid);
    ko_swiglu(m->w1_out, m->w3_out, m->w1_out, hid);
    linear_forward(m, &m->w2[l], m->w1_out, m->rms_out, hid, dim);
    ko_add(m->x, m->rms_out, m->x, dim);
  }
  /* cls_logits :722-731 (final norm in place) */
  ko_rmsnorm(m->x, m->final_norm, m->x, dim, eps);
  linear_forward(m, &m->wcls, m->x, m->logits, dim, c->vocab_size);
  if (logits_out) memcpy(logits_out, m->logits, sizeof(float) * c->vocab_size);
  return (int)ko_argmax(m->logits, c->vocab_size);
}
