/*
 * lnb_oracle.h -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE)
 *
 * A plain-C restatement of the arithmetic of adalkiran/llama-nuts-and-bolts'
 * Llama-3.1 forward path (Go, CPU).  Every function cites the reference
 * file:line it follows (paths relative to the reference repo root).
 *
 * Who may use this: tests/, __graft_entry__.smoke(), and bench.py's
 * cpu_baseline / --impl reference legs.  The product (liblnb.so and the
 * llama-nuts-and-bolts_b200 package) never links, imports or calls it.
 *
 * Parity status: PINNED.  The restatement reproduces the reference's own
 * weight-free golden vectors (src/dtype/bfloat16_test.go, src/ml/operations_test.go
 * Linear/MatMul/Pow/Mean, docs/10-ROPE...md frequency table); see
 * tests/test_oracle_golden.py.  The Go toolchain is absent in this image, so the
 * reference itself cannot be executed here (DESIGN.md "Oracle").
 *
 * Numeric model (SURVEY.md Appendix A): t(x) = f32 -> bf16 by TRUNCATION
 * (bits >> 16, src/dtype/bfloat16.go:31-33,59-61); every op reads bf16 as f32,
 * computes in f32 (a few steps in f64) and truncates its result; all sums are
 * strictly sequential in increasing index order with one f32 rounding per add.
 * Compile with -ffp-contract=off (Go/amd64 never fuses x*y+z).
 */
#ifndef LNB_ORACLE_H
#define LNB_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- src/dtype/bfloat16.go:19-21,31-33,55-61 ---- */
uint16_t orc_f32_to_bf16(float f);
float    orc_bf16_to_f32(uint16_t b);

/* ---- src/ml ops (each returns 0 on success) ---- */
/* ml.LinearTransformation BF16: operations_lineartransform.go:37-70,145-207.
 * x[S,K] bf16, w[N,K] bf16 -> out[S,N] bf16 = t(sum_seq_k x*w). */
void orc_linear_bf16(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int K, int N);
/* same sums, untruncated f32 result (used to build TP / split-K expectations) */
void orc_linear_bf16_f32out(const uint16_t* x, const uint16_t* w, float* out, int S, int K, int N);
/* ml.LinearTransformation F32: operations_lineartransform.go:72-103 */
void orc_linear_f32(const float* x, const float* w, float* out, int S, int K, int N);
/* ml.MatMul BF16: operations_matmul.go:24-60,136-182. a[B,M,K] x b[B,K,N] -> out[B,M,N] */
void orc_matmul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int B, int M, int K, int N);
/* ml.Pow(x,2) on bf16 -> f32: operations_impl.go:197-217 */
void orc_pow2_bf16(const uint16_t* x, float* out, int64_t n);
/* ml.Mean(dim=-1) on f32: operations_impl.go:219-253 */
void orc_mean_f32(const float* x, float* out, int rows, int cols);
/* ml.Add / ml.MultiplyElementwise on bf16 (same shape): operations_impl.go:307-335,367-395 */
void orc_add_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n);
void orc_mul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n);
/* ml.DivToScalar on bf16 with a bf16 scalar: operations_impl.go:273-289 */
void orc_div_scalar_bf16(const uint16_t* a, uint16_t scalar_bf16, uint16_t* out, int64_t n);
/* ml.Softmax on f32 rows (f64 exp/sum, no max subtraction): operations_impl.go:478-511 */
void orc_softmax_f32(const float* x, float* out, int rows, int cols);
/* ml.Argmax last dim (strict '<', first max wins): operations_impl.go:513-548 */
int32_t orc_argmax_f32(const float* x, int n);
/* ml.Silu on bf16 via the 65536-entry table: activations.go:11-50 */
void orc_silu_bf16(const uint16_t* x, uint16_t* out, int64_t n);
/* the table itself, already truncated to bf16: out[65536] */
void orc_silu_table_bf16(uint16_t* out);
/* ml.Fwd_Get_Rows: operations_impl.go:142-173 */
void orc_get_rows_bf16(const uint16_t* emb, const int32_t* tokens, uint16_t* out, int S, int dim);

/* ---- src/model pieces ---- */
/* RMSNorm.doNormalization (stage 1 only): llamatransformer.go:641-660 */
void orc_rms_scale(const uint16_t* x, float* r, int S, int D, float eps);
void orc_rmsnorm_stage1(const uint16_t* x, uint16_t* out, int S, int D, float eps);
/* RMSNorm.Forward: llamatransformer.go:633-639 */
void orc_rmsnorm(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int D, float eps);
/* precomputeFreqsCis + applyScaling: llamatransformer.go:662-751.
 * freqs_out (optional) [dim/2] bf16 scaled inverse frequencies;
 * cis_out [end][dim/2][2] f32 (cos, sin) == complex64 table. */
void orc_rope_table(int dim, int end, double theta, int use_scaled, uint16_t* freqs_out, float* cis_out);
/* applyRotaryEmbeddings for one tensor x[S,H,hd] bf16 with table rows
 * [start_pos, start_pos+S): llamatransformer.go:753-790, operations_impl.go:396-423
 * (Go complex64 multiply is evaluated through float64 intermediates). */
void orc_rope_apply(const uint16_t* x, const float* cis, uint16_t* out, int S, int H, int hd, int start_pos);
/* scaled-dot-product attention over cache rows [0,T): llamatransformer.go:402-514.
 * q[S,n_heads,hd] (already rotated), cacheK/V [>=T, n_kv, hd]; out [S, n_heads*hd]. */
void orc_attention(const uint16_t* q, const uint16_t* cacheK, const uint16_t* cacheV, uint16_t* out,
                   int S, int T, int n_heads, int n_kv, int hd, int causal_mask);
/* extension (beyond the reference): the same with query row s at absolute position q_pos0 + s, so a causal row sees the
 * keys t <= q_pos0 + s -- the [S,T] mask of a chunked prefill (q_pos0 = T - S) */
void orc_attention_pos(const uint16_t* q, const uint16_t* cacheK, const uint16_t* cacheV, uint16_t* out,
                       int S, int T, int n_heads, int n_kv, int hd, int causal_mask, int q_pos0);

/* ---- whole model ---- */
typedef struct {
  int dim, n_layers, n_heads, n_kv_heads, head_dim, ffn_dim, vocab, max_seq_len;
  float norm_eps;
  double rope_theta;
  int use_scaled_rope;
} orc_args;

typedef struct orc_model orc_model;
typedef struct orc_session orc_session;

orc_model*  orc_model_new(const orc_args* a);
void        orc_model_free(orc_model* m);
/* Bind a tensor by its checkpoint name ("layers.3.attention.wq.weight", ...).
 * The pointer is BORROWED (mirrors the reference's mmap-aliasing tensors,
 * src/torch/types.go:51-56).  Returns 0, or -1 for an unknown name. */
int         orc_model_bind(orc_model* m, const char* name, const uint16_t* data);
orc_session* orc_session_new(const orc_model* m, int seq_len);   /* inferencecontext.go:17-46 */
void        orc_session_free(orc_session* s);
uint16_t*   orc_session_cache_k(orc_session* s, int layer);
uint16_t*   orc_session_cache_v(orc_session* s, int layer);
/* LlamaTransformer.Forward: llamatransformer.go:145-180.
 * logits: [S,vocab] f32 if all_rows, else [1,vocab] (last row only).
 * trace (optional): residual stream after each layer, [(n_layers+1)][S][dim] bf16
 * (slot 0 = embeddings).  Returns 0 or -1. */
int         orc_forward(const orc_model* m, orc_session* s, const int32_t* tokens, int S, int start_pos,
                        float* logits, int all_rows, uint16_t* trace);
/* variant that emulates tensor-parallel K-split partial sums:
 * wo and w2 are accumulated as `tp` sequential partial sums over contiguous K
 * slices which are then added in rank order 0..tp-1 (f32) before truncation. */
/* extension (beyond the reference): S > 1 tokens at start_pos > 0 with the [S,T] causal mask -- chunked prefill */
int         orc_forward_chunk(const orc_model* m, orc_session* s, const int32_t* tokens, int S, int start_pos,
                              float* logits, int all_rows);
int         orc_forward_tp(const orc_model* m, orc_session* s, const int32_t* tokens, int S, int start_pos,
                           float* logits, int all_rows, int tp);
/* generateTokensInternal: src/inference/inference.go:173-254.  Returns number of
 * generated tokens written to out (prompt tokens are not copied). */
int         orc_generate(const orc_model* m, const int32_t* prompt, int n_prompt, int seq_len,
                         const int32_t* stop_ids, int n_stop, int32_t* out, double* step_seconds);

/* ---- synthetic checkpoint (SURVEY.md 8d; not from the reference) ---- */
/* value(i) = t( (2u-1)*scale + offset ), u = top 24 bits of splitmix64(seed ^ fnv1a(name), i) */
void orc_synth_fill(uint64_t seed, const char* name, float scale, float offset, int64_t n, uint16_t* out);

int  orc_num_threads(void);
void orc_set_num_threads(int n);

#ifdef __cplusplus
}
#endif
#endif
