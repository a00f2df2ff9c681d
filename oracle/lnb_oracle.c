/*
 * lnb_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 * See lnb_oracle.h for scope, parity status and the numeric model.
 * Build: oracle/Makefile  (gcc -O3 -ffp-contract=off -fopenmp).
 *
 * Parallelism mirrors the reference's goroutine fan-out: over output rows /
 * output features only, never over the reduction index k
 * (src/ml/operations_lineartransform.go:119-130,173-184).
 */
#include "lnb_oracle.h"
#include <math.h>
#include <omp.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------ dtype */

static inline float bf(uint16_t b) {
  uint32_t u = (uint32_t)b << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static inline uint16_t tr(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return (uint16_t)(u >> 16);
}
uint16_t orc_f32_to_bf16(float f) { return tr(f); }
float orc_bf16_to_f32(uint16_t b) { return bf(b); }

int orc_num_threads(void) { return omp_get_max_threads(); }
void orc_set_num_threads(int n) {
  if (n > 0) omp_set_num_threads(n);
}

/* ----------------------------------------------------------------- linear */

/* One output feature, S==1: strictly sequential k, f32 accumulate
 * (operations_lineartransform.go:45-69).  Eight independent outputs are
 * processed side by side (one per SIMD lane / scalar chain) only to give the
 * CPU independent dependency chains; each output still sees k = 0,1,2,... */
#if defined(__AVX2__)
#include <immintrin.h>
static inline __m256 bf8_to_f32(const uint16_t* p) {
  __m128i h = _mm_loadu_si128((const __m128i*)p);
  return _mm256_castsi256_ps(_mm256_slli_epi32(_mm256_cvtepu16_epi32(h), 16));
}
static inline void transpose8(__m256* r) {
  __m256 t0 = _mm256_unpacklo_ps(r[0], r[1]), t1 = _mm256_unpackhi_ps(r[0], r[1]);
  __m256 t2 = _mm256_unpacklo_ps(r[2], r[3]), t3 = _mm256_unpackhi_ps(r[2], r[3]);
  __m256 t4 = _mm256_unpacklo_ps(r[4], r[5]), t5 = _mm256_unpackhi_ps(r[4], r[5]);
  __m256 t6 = _mm256_unpacklo_ps(r[6], r[7]), t7 = _mm256_unpackhi_ps(r[6], r[7]);
  __m256 u0 = _mm256_shuffle_ps(t0, t2, 0x44), u1 = _mm256_shuffle_ps(t0, t2, 0xEE);
  __m256 u2 = _mm256_shuffle_ps(t1, t3, 0x44), u3 = _mm256_shuffle_ps(t1, t3, 0xEE);
  __m256 u4 = _mm256_shuffle_ps(t4, t6, 0x44), u5 = _mm256_shuffle_ps(t4, t6, 0xEE);
  __m256 u6 = _mm256_shuffle_ps(t5, t7, 0x44), u7 = _mm256_shuffle_ps(t5, t7, 0xEE);
  r[0] = _mm256_permute2f128_ps(u0, u4, 0x20); r[1] = _mm256_permute2f128_ps(u1, u5, 0x20);
  r[2] = _mm256_permute2f128_ps(u2, u6, 0x20); r[3] = _mm256_permute2f128_ps(u3, u7, 0x20);
  r[4] = _mm256_permute2f128_ps(u0, u4, 0x31); r[5] = _mm256_permute2f128_ps(u1, u5, 0x31);
  r[6] = _mm256_permute2f128_ps(u2, u6, 0x31); r[7] = _mm256_permute2f128_ps(u3, u7, 0x31);
}
#endif

static void linear_s1(const float* xf, const uint16_t* w, float* accout, int K, int N, int kbeg, int kend) {
#pragma omp parallel for schedule(static)
  for (int nb = 0; nb < (N + 7) / 8; nb++) {
    int n0 = nb * 8, cnt = N - n0 < 8 ? N - n0 : 8;
    const uint16_t* wr[8];
    for (int j = 0; j < 8; j++) wr[j] = w + (size_t)(n0 + (j < cnt ? j : 0)) * K;
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int k = kbeg;
#if defined(__AVX2__)
    __m256 acc = _mm256_setzero_ps(); /* lane j = output n0+j */
    for (; k + 8 <= kend; k += 8) {
      __m256 r[8];
      for (int j = 0; j < 8; j++) r[j] = bf8_to_f32(wr[j] + k);
      transpose8(r); /* r[kk] lane j = w[n0+j][k+kk] */
      for (int kk = 0; kk < 8; kk++) {
        __m256 p = _mm256_mul_ps(_mm256_set1_ps(xf[k + kk]), r[kk]); /* exact product */
        acc = _mm256_add_ps(acc, p);                                  /* one rounding per add */
      }
    }
    _mm256_storeu_ps(a, acc);
#endif
    for (; k < kend; k++) {
      float xv = xf[k];
      for (int j = 0; j < 8; j++) a[j] += xv * bf(wr[j][k]);
    }
    for (int j = 0; j < cnt; j++) accout[n0 + j] = a[j];
  }
}

#define SB 16
/* S>1: input rows are transposed in blocks of SB so that the SB independent
 * per-row chains of one output feature sit in SIMD lanes.  Each lane still
 * performs the reference's sequential k loop. */
static void linear_sN(const uint16_t* x, const uint16_t* w, float* accout /*[S][N]*/, int S, int K, int N,
                      int kbeg, int kend) {
  int nblk = (S + SB - 1) / SB;
  float* xT = (float*)malloc((size_t)nblk * K * SB * sizeof(float));
  for (int b = 0; b < nblk; b++)
    for (int k = 0; k < K; k++)
      for (int j = 0; j < SB; j++) {
        int s = b * SB + j;
        xT[((size_t)b * K + k) * SB + j] = s < S ? bf(x[(size_t)s * K + k]) : 0.0f;
      }
#pragma omp parallel for schedule(static)
  for (int n = 0; n < N; n++) {
    const uint16_t* wr = w + (size_t)n * K;
    for (int b = 0; b < nblk; b++) {
      float a[SB];
      for (int j = 0; j < SB; j++) a[j] = 0.0f;
      const float* xb = xT + (size_t)b * K * SB;
      for (int k = kbeg; k < kend; k++) {
        float wv = bf(wr[k]);
        const float* xr = xb + (size_t)k * SB;
#pragma omp simd
        for (int j = 0; j < SB; j++) a[j] += xr[j] * wv;
      }
      for (int j = 0; j < SB; j++) {
        int s = b * SB + j;
        if (s < S) accout[(size_t)s * N + n] = a[j];
      }
    }
  }
  free(xT);
}

static void linear_acc(const uint16_t* x, const uint16_t* w, float* acc, int S, int K, int N, int kbeg, int kend) {
  if (S == 1) {
    float* xf = (float*)malloc((size_t)K * sizeof(float));
    for (int k = 0; k < K; k++) xf[k] = bf(x[k]);
    linear_s1(xf, w, acc, K, N, kbeg, kend);
    free(xf);
  } else {
    linear_sN(x, w, acc, S, K, N, kbeg, kend);
  }
}

void orc_linear_bf16_f32out(const uint16_t* x, const uint16_t* w, float* out, int S, int K, int N) {
  linear_acc(x, w, out, S, K, N, 0, K);
}

void orc_linear_bf16(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int K, int N) {
  float* acc = (float*)malloc((size_t)S * N * sizeof(float));
  linear_acc(x, w, acc, S, K, N, 0, K);
  for (size_t i = 0; i < (size_t)S * N; i++) out[i] = tr(acc[i]); /* ToBFloat16, :205 */
  free(acc);
}

/* K split into `tp` contiguous slices, partials added in rank order (TP emulation) */
static void linear_bf16_ksplit(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int K, int N, int tp) {
  size_t n = (size_t)S * N;
  float* tot = (float*)malloc(n * sizeof(float));
  float* part = (float*)malloc(n * sizeof(float));
  int ks = K / tp;
  for (int r = 0; r < tp; r++) {
    linear_acc(x, w, r == 0 ? tot : part, S, K, N, r * ks, r == tp - 1 ? K : (r + 1) * ks);
    if (r > 0)
      for (size_t i = 0; i < n; i++) tot[i] = tot[i] + part[i];
  }
  for (size_t i = 0; i < n; i++) out[i] = tr(tot[i]);
  free(tot);
  free(part);
}

/* operations_lineartransform.go:72-103 (F32 flavour: same loop on float32 data) */
void orc_linear_f32(const float* x, const float* w, float* out, int S, int K, int N) {
  for (int s = 0; s < S; s++)
    for (int n = 0; n < N; n++) {
      float a = 0.0f;
      for (int k = 0; k < K; k++) a += x[(size_t)s * K + k] * w[(size_t)n * K + k];
      out[(size_t)s * N + n] = a;
    }
}

/* operations_matmul.go:33-59 (strided column read of `other`), :160-182 */
void orc_matmul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int B, int M, int K, int N) {
#pragma omp parallel for collapse(2) schedule(static)
  for (int g = 0; g < B; g++)
    for (int m = 0; m < M; m++) {
      const uint16_t* ar = a + ((size_t)g * M + m) * K;
      const uint16_t* bg = b + (size_t)g * K * N;
      for (int n = 0; n < N; n++) {
        float acc = 0.0f;
        for (int k = 0; k < K; k++) acc += bf(ar[k]) * bf(bg[(size_t)k * N + n]);
        out[((size_t)g * M + m) * N + n] = tr(acc);
      }
    }
}

/* -------------------------------------------------------- elementwise ops */

void orc_pow2_bf16(const uint16_t* x, float* out, int64_t n) {
  /* float32(math.Pow(float64(x), 2)) -- x*x is exact in f64 (operations_impl.go:213) */
  for (int64_t i = 0; i < n; i++) {
    double v = (double)bf(x[i]);
    out[i] = (float)(v * v);
  }
}

void orc_mean_f32(const float* x, float* out, int rows, int cols) {
  for (int r = 0; r < rows; r++) {
    float s = 0.0f;
    for (int c = 0; c < cols; c++) s += x[(size_t)r * cols + c]; /* :238-244 */
    out[r] = s / (float)cols;                                    /* :246 */
  }
}

void orc_add_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n) {
  for (int64_t i = 0; i < n; i++) out[i] = tr(bf(a[i]) + bf(b[i]));
}
void orc_mul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n) {
  for (int64_t i = 0; i < n; i++) out[i] = tr(bf(a[i]) * bf(b[i]));
}
void orc_div_scalar_bf16(const uint16_t* a, uint16_t scalar_bf16, uint16_t* out, int64_t n) {
  float sc = bf(scalar_bf16);
  for (int64_t i = 0; i < n; i++) out[i] = tr(bf(a[i]) / sc);
}

void orc_softmax_f32(const float* x, float* out, int rows, int cols) {
  for (int r = 0; r < rows; r++) {
    const float* xr = x + (size_t)r * cols;
    double z = 0.0;
    for (int c = 0; c < cols; c++) z += exp((double)xr[c]); /* :492-498 */
    for (int c = 0; c < cols; c++) out[(size_t)r * cols + c] = (float)(exp((double)xr[c]) / z); /* :501-507 */
  }
}

int32_t orc_argmax_f32(const float* x, int n) {
  float maxv = -3.40282346638528859811704183484516925440e+38f; /* -math.MaxFloat32 */
  int32_t idx = -1;
  for (int i = 0; i < n; i++)
    if (maxv < x[i]) { /* strict '<': lowest index wins ties; NaN never selected */
      maxv = x[i];
      idx = i;
    }
  return idx;
}

static uint16_t g_silu_tab[65536];
static int g_silu_ready = 0;
static void silu_init(void) {
  if (g_silu_ready) return;
  for (int i = 0; i < 65536; i++) {
    double v = (double)bf((uint16_t)i);
    float s = (float)(v / (1.0 + exp(-v))); /* activations.go:22-25 */
    g_silu_tab[i] = tr(s);                  /* BFloat16fromFloat32(TABLE_SILU[bits]) :38 */
  }
  g_silu_ready = 1;
}
void orc_silu_table_bf16(uint16_t* out) {
  silu_init();
  memcpy(out, g_silu_tab, sizeof(g_silu_tab));
}
void orc_silu_bf16(const uint16_t* x, uint16_t* out, int64_t n) {
  silu_init();
  for (int64_t i = 0; i < n; i++) out[i] = g_silu_tab[x[i]];
}

void orc_get_rows_bf16(const uint16_t* emb, const int32_t* tokens, uint16_t* out, int S, int dim) {
  for (int s = 0; s < S; s++) memcpy(out + (size_t)s * dim, emb + (size_t)tokens[s] * dim, (size_t)dim * 2);
}

/* ---------------------------------------------------------------- RMSNorm */

static float rms_scale(const uint16_t* xr, int D, float eps) {
  float sum = 0.0f;
  for (int j = 0; j < D; j++) {
    double v = (double)bf(xr[j]);
    sum += (float)(v * v); /* Pow -> f32, then Mean's sequential f32 sum */
  }
  float mean = sum / (float)D;
  float me = mean + eps;                      /* AddScalar, f32 */
  return (float)(1.0 / sqrt((double)me));     /* RSqrt :300 */
}

/* the scale alone (llamatransformer.go:641-656), for white-box checks of the GPU scale kernels */
void orc_rms_scale(const uint16_t* x, float* r, int S, int D, float eps) {
  for (int s = 0; s < S; s++) r[s] = rms_scale(x + (size_t)s * D, D, eps);
}

void orc_rmsnorm_stage1(const uint16_t* x, uint16_t* out, int S, int D, float eps) {
  for (int s = 0; s < S; s++) {
    const uint16_t* xr = x + (size_t)s * D;
    float r = rms_scale(xr, D, eps);
    for (int j = 0; j < D; j++) out[(size_t)s * D + j] = tr(bf(xr[j]) * r); /* MultiplyElementwise(x,h) -> bf16 */
  }
}

void orc_rmsnorm(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int D, float eps) {
  for (int s = 0; s < S; s++) {
    const uint16_t* xr = x + (size_t)s * D;
    float r = rms_scale(xr, D, eps);
    for (int j = 0; j < D; j++) {
      uint16_t n1 = tr(bf(xr[j]) * r);
      out[(size_t)s * D + j] = tr(bf(n1) * bf(w[j])); /* llamatransformer.go:638 */
    }
  }
}

/* ------------------------------------------------------------------- RoPE */

void orc_rope_table(int dim, int end, double theta, int use_scaled, uint16_t* freqs_out, float* cis_out) {
  int half = dim / 2;
  uint16_t* freqs = (uint16_t*)malloc((size_t)half * 2);
  float dimf = (float)dim;
  for (int i = 0; i < half; i++) {
    float val = bf(tr((float)(2 * i)));                       /* ARange(0,dim,2,BF16) :713 */
    float f = (float)(1.0 / pow(theta, (double)(val / dimf))); /* :717-719 */
    freqs[i] = tr(f);                                         /* Apply_AsFloat32 writes bf16 */
  }
  if (use_scaled) { /* applyScaling :662-692, all float32 */
    const float scaleFactor = 8.0f, lowFreqFactor = 1.0f, highFreqFactor = 4.0f, oldContextLen = 8192.0f;
    const float lowFreqWavelen = oldContextLen / lowFreqFactor;
    const float highFreqWavelen = oldContextLen / highFreqFactor;
    const float twoPi = (float)(2.0 * 3.14159265358979323846264338327950288);
    for (int i = 0; i < half; i++) {
      float freq = bf(freqs[i]);
      float newFreq;
      float wavelen = twoPi / freq;
      if (wavelen < highFreqWavelen) {
        newFreq = freq;
      } else if (wavelen > lowFreqWavelen) {
        newFreq = freq / scaleFactor;
      } else {
        float smooth = (oldContextLen / wavelen - lowFreqFactor) / (highFreqFactor - lowFreqFactor);
        float t1 = (1.0f - smooth) * freq;
        t1 = t1 / scaleFactor;
        float t2 = smooth * freq;
        newFreq = t1 + t2;
      }
      freqs[i] = tr(newFreq);
    }
  }
  if (freqs_out) memcpy(freqs_out, freqs, (size_t)half * 2);
  if (cis_out) {
    for (int p = 0; p < end; p++) {
      float tp = bf(tr((float)p)); /* ARange(0,end,1,BF16): positions quantised to bf16 :724 */
      for (int i = 0; i < half; i++) {
        float ang = bf(tr(tp * bf(freqs[i])));       /* Outer -> bf16, operations_impl.go:47-48 */
        double a64 = (double)ang;
        double re = 1.0 * cos(a64), im = 1.0 * sin(a64); /* Polar :131-133 */
        cis_out[((size_t)p * half + i) * 2 + 0] = (float)re;
        cis_out[((size_t)p * half + i) * 2 + 1] = (float)im;
      }
    }
  }
  free(freqs);
}

void orc_rope_apply(const uint16_t* x, const float* cis, uint16_t* out, int S, int H, int hd, int start_pos) {
  int half = hd / 2;
  for (int s = 0; s < S; s++)
    for (int h = 0; h < H; h++)
      for (int i = 0; i < half; i++) {
        size_t o = ((size_t)s * H + h) * hd + 2 * i;
        double a = (double)bf(x[o]), b = (double)bf(x[o + 1]);
        const float* fc = cis + ((size_t)(start_pos + s) * half + i) * 2;
        double c = (double)fc[0], d = (double)fc[1];
        /* Go gc lowers complex64*complex64 through float64 (SURVEY F16-A1) */
        float re = (float)(a * c - b * d);
        float im = (float)(a * d + b * c);
        out[o] = tr(re);
        out[o + 1] = tr(im);
      }
}

/* -------------------------------------------------------------- attention */

/* q_pos0 = absolute position of query row 0.  The reference only ever builds the [S,S] mask for startPos 0 (T == S,
 * q_pos0 = 0: `t > s`, llamatransformer.go:128-136); q_pos0 > 0 is the chunked-prefill EXTENSION (beyond the reference):
 * the [S,T] mask a correct broadcast would need, row s sees the keys t <= q_pos0 + s. */
static void attention_impl(const uint16_t* q, const uint16_t* cacheK, const uint16_t* cacheV, uint16_t* out, int S, int T,
                           int n_heads, int n_kv, int hd, int causal_mask, int q_pos0) {
  int n_rep = n_heads / n_kv;
  /* dtype.BFloat16fromFloat32(float32(math.Sqrt(float64(HeadDim)))) llamatransformer.go:464 */
  float scale = bf(tr((float)sqrt((double)hd)));
  float ninf = -INFINITY;
#pragma omp parallel for collapse(2) schedule(static)
  for (int s = 0; s < S; s++)
    for (int H = 0; H < n_heads; H++) {
      int h = H / n_rep; /* attentionRepeatKV :529-559: expanded head H <- kv head H / N_Rep */
      const uint16_t* qr = q + ((size_t)s * n_heads + H) * hd;
      uint16_t* sc = (uint16_t*)malloc((size_t)T * 2);
      double* e = (double*)malloc((size_t)T * sizeof(double));
      for (int t = 0; t < T; t++) {
        const uint16_t* kr = cacheK + ((size_t)t * n_kv + h) * hd;
        float acc = 0.0f;
        for (int d = 0; d < hd; d++) acc += bf(qr[d]) * bf(kr[d]); /* MatMul(xq, keys^T) :459 */
        uint16_t v = tr(acc);
        v = tr(bf(v) / scale);                                     /* DivToScalar :464 */
        if (causal_mask) {
          float mk = (t > s + q_pos0) ? ninf : 0.0f;               /* triu(full(-inf),1) :128-136 */
          v = tr(bf(v) + mk);                                      /* Add(scores, mask) :471 */
        }
        sc[t] = v;
      }
      double z = 0.0;
      for (int t = 0; t < T; t++) {
        e[t] = exp((double)bf(sc[t])); /* ToFloat32 -> Softmax (f64, no max-subtraction) :484-490 */
        z += e[t];
      }
      for (int t = 0; t < T; t++) sc[t] = tr((float)(e[t] / z)); /* -> f32 -> ToBFloat16 :493 */
      uint16_t* orow = out + (size_t)s * n_heads * hd + (size_t)H * hd; /* Transpose(0,1)+Reshape :508-514 */
      for (int d = 0; d < hd; d++) {
        float acc = 0.0f;
        for (int t = 0; t < T; t++) acc += bf(sc[t]) * bf(cacheV[((size_t)t * n_kv + h) * hd + d]); /* :504 */
        orow[d] = tr(acc);
      }
      free(sc);
      free(e);
    }
}

void orc_attention(const uint16_t* q, const uint16_t* cacheK, const uint16_t* cacheV, uint16_t* out, int S, int T,
                   int n_heads, int n_kv, int hd, int causal_mask) {
  attention_impl(q, cacheK, cacheV, out, S, T, n_heads, n_kv, hd, causal_mask, 0);
}

void orc_attention_pos(const uint16_t* q, const uint16_t* cacheK, const uint16_t* cacheV, uint16_t* out, int S, int T,
                       int n_heads, int n_kv, int hd, int causal_mask, int q_pos0) {
  attention_impl(q, cacheK, cacheV, out, S, T, n_heads, n_kv, hd, causal_mask, q_pos0);
}

/* ------------------------------------------------------------ whole model */

struct orc_model {
  orc_args a;
  const uint16_t *tok_embd, *norm, *output;
  const uint16_t **attn_norm, **wq, **wk, **wv, **wo, **ffn_norm, **w1, **w2, **w3;
  float* cis; /* [2*max_seq_len][head_dim/2][2] */
};

struct orc_session {
  const orc_model* m;
  int seq_len;
  uint16_t **ck, **cv;
};

orc_model* orc_model_new(const orc_args* a) {
  orc_model* m = (orc_model*)calloc(1, sizeof(orc_model));
  m->a = *a;
  int L = a->n_layers;
  const uint16_t*** arrs[] = {&m->attn_norm, &m->wq, &m->wk, &m->wv, &m->wo, &m->ffn_norm, &m->w1, &m->w2, &m->w3};
  for (unsigned i = 0; i < sizeof(arrs) / sizeof(arrs[0]); i++) *arrs[i] = (const uint16_t**)calloc(L, sizeof(void*));
  int end = a->max_seq_len * 2; /* llamatransformer.go:109 */
  m->cis = (float*)malloc((size_t)end * (a->head_dim / 2) * 2 * sizeof(float));
  orc_rope_table(a->head_dim, end, a->rope_theta, a->use_scaled_rope, NULL, m->cis);
  silu_init();
  return m;
}

void orc_model_free(orc_model* m) {
  if (!m) return;
  free(m->attn_norm); free(m->wq); free(m->wk); free(m->wv); free(m->wo);
  free(m->ffn_norm); free(m->w1); free(m->w2); free(m->w3); free(m->cis);
  free(m);
}

int orc_model_bind(orc_model* m, const char* name, const uint16_t* data) {
  if (!strcmp(name, "tok_embeddings.weight")) { m->tok_embd = data; return 0; }
  if (!strcmp(name, "norm.weight")) { m->norm = data; return 0; }
  if (!strcmp(name, "output.weight")) { m->output = data; return 0; }
  int l = -1;
  char rest[96];
  if (sscanf(name, "layers.%d.%95s", &l, rest) != 2 || l < 0 || l >= m->a.n_layers) return -1;
  if (!strcmp(rest, "attention_norm.weight")) m->attn_norm[l] = data;
  else if (!strcmp(rest, "attention.wq.weight")) m->wq[l] = data;
  else if (!strcmp(rest, "attention.wk.weight")) m->wk[l] = data;
  else if (!strcmp(rest, "attention.wv.weight")) m->wv[l] = data;
  else if (!strcmp(rest, "attention.wo.weight")) m->wo[l] = data;
  else if (!strcmp(rest, "ffn_norm.weight")) m->ffn_norm[l] = data;
  else if (!strcmp(rest, "feed_forward.w1.weight")) m->w1[l] = data;
  else if (!strcmp(rest, "feed_forward.w2.weight")) m->w2[l] = data;
  else if (!strcmp(rest, "feed_forward.w3.weight")) m->w3[l] = data;
  else return -1;
  return 0;
}

orc_session* orc_session_new(const orc_model* m, int seq_len) {
  orc_session* s = (orc_session*)calloc(1, sizeof(orc_session));
  s->m = m;
  s->seq_len = seq_len;
  int L = m->a.n_layers;
  size_t n = (size_t)seq_len * m->a.n_kv_heads * m->a.head_dim;
  s->ck = (uint16_t**)calloc(L, sizeof(void*));
  s->cv = (uint16_t**)calloc(L, sizeof(void*));
  for (int l = 0; l < L; l++) {
    s->ck[l] = (uint16_t*)calloc(n, 2); /* ml.Zeros, inferencecontext.go:31-43 */
    s->cv[l] = (uint16_t*)calloc(n, 2);
  }
  return s;
}
void orc_session_free(orc_session* s) {
  if (!s) return;
  for (int l = 0; l < s->m->a.n_layers; l++) { free(s->ck[l]); free(s->cv[l]); }
  free(s->ck); free(s->cv); free(s);
}
uint16_t* orc_session_cache_k(orc_session* s, int layer) { return s->ck[layer]; }
uint16_t* orc_session_cache_v(orc_session* s, int layer) { return s->cv[layer]; }

static int g_allow_chunk = 0; /* set only inside orc_forward_chunk (extension) */
static int forward_impl(const orc_model* m, orc_session* ss, const int32_t* tokens, int S, int start_pos,
                        float* logits, int all_rows, uint16_t* trace, int tp) {
  const orc_args* a = &m->a;
  if (S <= 0) return -1; /* "empty token array" llamatransformer.go:146-148 */
  if (start_pos + S > ss->seq_len) return -1;
  if (S > 1 && start_pos != 0 && !g_allow_chunk) return -1; /* mask [S,S] only broadcasts when T==S (SURVEY F11) */
  int D = a->dim, hd = a->head_dim, nh = a->n_heads, nkv = a->n_kv_heads, F = a->ffn_dim, V = a->vocab;
  int kvd = nkv * hd, qd = nh * hd;
  for (int s = 0; s < S; s++)
    if (tokens[s] < 0 || tokens[s] >= V) return -1;
  size_t SD = (size_t)S * D;
  uint16_t* x = (uint16_t*)malloc(SD * 2);
  uint16_t* xn = (uint16_t*)malloc(SD * 2);
  uint16_t* q = (uint16_t*)malloc((size_t)S * qd * 2);
  uint16_t* q2 = (uint16_t*)malloc((size_t)S * qd * 2);
  uint16_t* k = (uint16_t*)malloc((size_t)S * kvd * 2);
  uint16_t* k2 = (uint16_t*)malloc((size_t)S * kvd * 2);
  uint16_t* v = (uint16_t*)malloc((size_t)S * kvd * 2);
  uint16_t* o = (uint16_t*)malloc((size_t)S * qd * 2);
  uint16_t* att = (uint16_t*)malloc(SD * 2);
  uint16_t* h1 = (uint16_t*)malloc(SD * 2);
  uint16_t* g = (uint16_t*)malloc((size_t)S * F * 2);
  uint16_t* u = (uint16_t*)malloc((size_t)S * F * 2);
  uint16_t* ff = (uint16_t*)malloc(SD * 2);
  int T = start_pos + S;

  orc_get_rows_bf16(m->tok_embd, tokens, x, S, D); /* prepare :118 */
  if (trace) memcpy(trace, x, SD * 2);
  for (int l = 0; l < a->n_layers; l++) {
    orc_rmsnorm(x, m->attn_norm[l], xn, S, D, a->norm_eps);          /* :222 */
    orc_linear_bf16(xn, m->wq[l], q, S, D, qd);                      /* :306 */
    orc_linear_bf16(xn, m->wk[l], k, S, D, kvd);                     /* :325 */
    orc_linear_bf16(xn, m->wv[l], v, S, D, kvd);                     /* :344 */
    orc_rope_apply(q, m->cis, q2, S, nh, hd, start_pos);             /* :392 */
    orc_rope_apply(k, m->cis, k2, S, nkv, hd, start_pos);
    memcpy(ss->ck[l] + (size_t)start_pos * kvd, k2, (size_t)S * kvd * 2); /* SetSlice :402 */
    memcpy(ss->cv[l] + (size_t)start_pos * kvd, v, (size_t)S * kvd * 2);  /* :403 */
    attention_impl(q2, ss->ck[l], ss->cv[l], o, S, T, nh, nkv, hd, S > 1, start_pos); /* :409-514 (start_pos > 0: extension) */
    if (tp > 1) linear_bf16_ksplit(o, m->wo[l], att, S, qd, D, tp);
    else orc_linear_bf16(o, m->wo[l], att, S, qd, D);                /* :522 */
    orc_add_bf16(x, att, h1, (int64_t)SD);                           /* :232 */
    orc_rmsnorm(h1, m->ffn_norm[l], xn, S, D, a->norm_eps);          /* :237 */
    orc_linear_bf16(xn, m->w1[l], g, S, D, F);                       /* :601 */
    orc_silu_bf16(g, g, (int64_t)S * F);                             /* :605 */
    orc_linear_bf16(xn, m->w3[l], u, S, D, F);                       /* :610 */
    orc_mul_bf16(g, u, g, (int64_t)S * F);                           /* :614 */
    if (tp > 1) linear_bf16_ksplit(g, m->w2[l], ff, S, F, D, tp);
    else orc_linear_bf16(g, m->w2[l], ff, S, F, D);                  /* :619 */
    orc_add_bf16(h1, ff, x, (int64_t)SD);                            /* :248 */
    if (trace) memcpy(trace + (size_t)(l + 1) * SD, x, SD * 2);
  }
  orc_rmsnorm(x, m->norm, xn, S, D, a->norm_eps); /* :166 */
  if (logits) {
    int rows = all_rows ? S : 1;
    const uint16_t* src = all_rows ? xn : xn + (size_t)(S - 1) * D;
    uint16_t* lg = (uint16_t*)malloc((size_t)rows * V * 2);
    orc_linear_bf16(src, m->output, lg, rows, D, V);                 /* :170 */
    for (size_t i = 0; i < (size_t)rows * V; i++) logits[i] = bf(lg[i]); /* ToFloat32 :175 */
    free(lg);
  }
  free(x); free(xn); free(q); free(q2); free(k); free(k2); free(v); free(o); free(att); free(h1);
  free(g); free(u); free(ff);
  return 0;
}

int orc_forward(const orc_model* m, orc_session* s, const int32_t* tokens, int S, int start_pos, float* logits,
                int all_rows, uint16_t* trace) {
  return forward_impl(m, s, tokens, S, start_pos, logits, all_rows, trace, 1);
}
/* EXTENSION, beyond the reference: a prompt chunk of S > 1 tokens at start_pos > 0 (chunked prefill).  The reference
 * cannot do this (its [S,S] mask does not broadcast against [S,T] scores; the only caller prefills at 0).  Everything
 * but the mask's column offset is the reference's arithmetic, so prefilling a prompt in chunks gives bit-identical
 * results to prefilling it at once. */
int orc_forward_chunk(const orc_model* m, orc_session* s, const int32_t* tokens, int S, int start_pos, float* logits,
                      int all_rows) {
  g_allow_chunk = 1;
  int rc = forward_impl(m, s, tokens, S, start_pos, logits, all_rows, NULL, 1);
  g_allow_chunk = 0;
  return rc;
}
int orc_forward_tp(const orc_model* m, orc_session* s, const int32_t* tokens, int S, int start_pos, float* logits,
                   int all_rows, int tp) {
  return forward_impl(m, s, tokens, S, start_pos, logits, all_rows, NULL, tp);
}

static double now_s(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

int orc_generate(const orc_model* m, const int32_t* prompt, int n_prompt, int seq_len, const int32_t* stop_ids,
                 int n_stop, int32_t* out, double* step_seconds) {
  if (n_prompt >= seq_len) return -1; /* inference.go:176-179 */
  orc_session* s = orc_session_new(m, seq_len);
  int32_t* tokens = (int32_t*)malloc((size_t)seq_len * 4);
  for (int i = 0; i < seq_len; i++) tokens[i] = -1; /* PadId, :181 */
  for (int i = 0; i < n_prompt; i++) tokens[i] = prompt[i];
  float* logits = (float*)malloc((size_t)m->a.vocab * sizeof(float));
  int prev = 0, n_out = 0;
  for (int cur = n_prompt; cur < seq_len; cur++) { /* :194 */
    double t0 = now_s();
    if (orc_forward(m, s, tokens + prev, cur - prev, prev, logits, 0, NULL) != 0) { n_out = -1; break; }
    int32_t next = orc_argmax_f32(logits, m->a.vocab); /* :207-216 */
    if (tokens[cur] != -1) next = tokens[cur];         /* :218-226 */
    tokens[cur] = next;
    if (step_seconds) step_seconds[n_out] = now_s() - t0;
    out[n_out++] = next;
    prev = cur;
    int eos = 0;
    for (int i = 0; i < n_stop; i++) eos |= (stop_ids[i] == next);
    if (eos) break;                 /* :233-240 */
    if (cur + 1 == seq_len) break;  /* :241-247 */
  }
  free(tokens); free(logits);
  orc_session_free(s);
  return n_out;
}

/* ---------------------------------------------------- synthetic weights */

static inline uint64_t fnv1a64(const char* s) {
  uint64_t h = 0xcbf29ce484222325ULL;
  for (; *s; s++) { h ^= (uint8_t)*s; h *= 0x100000001b3ULL; }
  return h;
}
static inline uint64_t splitmix64_at(uint64_t seed, uint64_t i) {
  uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
void orc_synth_fill(uint64_t seed, const char* name, float scale, float offset, int64_t n, uint16_t* out) {
  uint64_t s = seed ^ fnv1a64(name);
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; i++) {
    uint64_t z = splitmix64_at(s, (uint64_t)i);
    float u = (float)(z >> 40) * (1.0f / 16777216.0f);
    float w = 2.0f * u - 1.0f;
    float v = w * scale;
    v = v + offset;
    out[i] = tr(v);
  }
}
