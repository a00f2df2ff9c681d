/* Sequential C statement of the seeded sampler (TEST INFRASTRUCTURE, NOT PRODUCT CODE; DESIGN.md §9b).
 *
 * The reference (inference.go:207-216) only has the greedy ml.Argmax, so sampling is an extension; this file states its
 * contract in the plainest form -- a full sort for the rank order, sequential integer sums -- for the tests to hold the
 * sampler kernel (csrc/sample.cuh) against.  The floating-point steps come from csrc/sample_det.h, the header the kernel
 * compiles too.  orc_generate_sampled drives the CPU oracle's forward (oracle/lnb_oracle.h) like orc_generate, with the
 * sampler in place of the argmax. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/lnb.h"
#include "../llama-nuts-and-bolts_b200/csrc/sample_det.h"
#include "../llama-nuts-and-bolts_b200/csrc/penalty_det.h"
#include "../oracle/lnb_oracle.h"

double orc_exp_det(double z) { return lnb_exp_det(z); }
void orc_exp_det_n(const double* z, double* out, int64_t n) {
  for (int64_t i = 0; i < n; i++) out[i] = lnb_exp_det(z[i]);
}
uint64_t orc_sample_weight(float l, float m, float T) { return lnb_sample_weight(l, m, T); }

/* max over the f32 values with bit patterns [lo, hi] (non-positive floats: 0x80000000 | magnitude bits) of the distance
 * in ulps between lnb_exp_det and libm's exp (the function Python's math.exp calls) */
int64_t orc_exp_det_max_ulp_f32(uint32_t lo, uint32_t hi) {
  int64_t worst = 0;
#pragma omp parallel for reduction(max : worst) schedule(static, 65536)
  for (int64_t b = lo; b <= (int64_t)hi; b++) {
    union { uint32_t u; float f; } c;
    c.u = (uint32_t)b;
    const double z = (double)c.f;
    const double a = lnb_exp_det(z), e = exp(z);
    int64_t ia, ie;
    memcpy(&ia, &a, 8);
    memcpy(&ie, &e, 8);
    const int64_t d = ia > ie ? ia - ie : ie - ia;   /* same sign, same binade or adjacent: bit distance = ulps */
    if (d > worst) worst = d;
  }
  return worst;
}

static const float* g_rank_l;
static int rank_cmp(const void* pa, const void* pb) {
  const int32_t a = *(const int32_t*)pa, b = *(const int32_t*)pb;
  const uint32_t ka = lnb_sample_ord(g_rank_l[a]), kb = lnb_sample_ord(g_rank_l[b]);
  if (ka != kb) return ka > kb ? -1 : 1;   /* logit descending */
  return a < b ? -1 : a > b ? 1 : 0;       /* then index ascending */
}

/* one row: the token id the contract draws (T == 0: the greedy argmax) */
int32_t orc_sample_row(const float* l, int V, float T, int32_t K, float P, uint64_t seed, int64_t p_next) {
  if (V <= 0) return -1;
  int32_t* order = (int32_t*)malloc((size_t)V * 4);
  for (int i = 0; i < V; i++) order[i] = i;
  g_rank_l = l;
  qsort(order, (size_t)V, 4, rank_cmp);
  if (T == 0.0f) {
    const int32_t t = order[0];
    free(order);
    return t;
  }
  const float m = l[order[0]];
  const int nC = (K == 0 || K >= V) ? V : K;           /* candidates: ranks < K */
  uint64_t* W = (uint64_t*)calloc((size_t)V, 8);       /* by index; 0 outside the kept set */
  uint64_t WC = 0;
  for (int r = 0; r < nC; r++) WC += lnb_sample_weight(l[order[r]], m, T);
  if (WC == 0) {                                       /* every weight 0 (top logit +inf or NaN): the rank-0 token */
    const int32_t t = order[0];
    free(W);
    free(order);
    return t;
  }
  int nkeep = nC;
  if (P < 1.0f) {                                      /* shortest rank prefix of C with mass >= Q */
    const uint64_t Q = lnb_sample_top_p_mass(P, WC);
    uint64_t acc = 0;
    for (int r = 0; r < nC; r++) {
      acc += lnb_sample_weight(l[order[r]], m, T);
      if (acc >= Q) { nkeep = r + 1; break; }
    }
  }
  uint64_t Wk = 0;
  for (int r = 0; r < nkeep; r++) {
    W[order[r]] = lnb_sample_weight(l[order[r]], m, T);
    Wk += W[order[r]];
  }
  const uint64_t R = lnb_sample_scale(lnb_splitmix64_at(seed, (uint64_t)p_next), Wk);
  int32_t tok = -1;
  uint64_t acc = 0;
  for (int i = 0; i < V; i++) {                        /* index order: smallest i whose prefix mass exceeds R */
    acc += W[i];
    if (acc > R) { tok = i; break; }
  }
  free(W);
  free(order);
  return tok;
}

/* one row: the log-probability record of token `target` (DESIGN.md §9d) -- a full sort for the ranks, a sequential sum of
 * the weights at temperature 1, then the shared host finish */
void orc_logprob_row(const float* l, int V, int32_t target, int top_n, lnb_logprob* out) {
  memset(out, 0, sizeof(*out));
  int32_t* order = (int32_t*)malloc((size_t)V * 4);
  for (int i = 0; i < V; i++) order[i] = i;
  g_rank_l = l;
  qsort(order, (size_t)V, 4, rank_cmp);
  const float m = l[order[0]];
  uint64_t sum = 0;
  for (int i = 0; i < V; i++) sum += lnb_sample_weight(l[i], m, 1.0f);
  int rank = 1;
  while (order[rank - 1] != target) rank++;
  out->token = target;
  out->rank = rank;
  out->logprob = lnb_logprob_finish(l[target], m, sum);
  out->n_top = top_n < V ? top_n : V;
  for (int r = 0; r < out->n_top; r++) {
    out->top_token[r] = order[r];
    out->top_logprob[r] = lnb_logprob_finish(l[order[r]], m, sum);
  }
  free(order);
}
void orc_logprob_rows(const float* l, int rows, int V, const int32_t* targets, int top_n, lnb_logprob* out) {
  for (int r = 0; r < rows; r++) orc_logprob_row(l + (size_t)r * V, V, targets[r], top_n, out + r);
}

/* one row: l' of the penalties and bias (DESIGN.md §9e) for the token at position p_next, given the tokens hist[0, p_next)
 * fed before it (-1: not counted) -- counts by a plain walk over the window, then the steps of csrc/penalty_det.h */
void orc_penalize_row(const float* l, int V, const lnb_penalties* p, const int32_t* hist, int32_t p_next, float* out) {
  if (lnb_pen_neutral(p)) {   /* off: the row itself */
    memcpy(out, l, (size_t)V * sizeof(float));
    return;
  }
  uint32_t* c = (uint32_t*)calloc((size_t)V, 4);
  int32_t lo = lnb_pen_lo(p, p_next);
  if (lo < 0) lo = 0;
  for (int32_t i = lo; i < p_next; i++)
    if (hist[i] >= 0 && hist[i] < V) c[hist[i]]++;
  for (int i = 0; i < V; i++) out[i] = lnb_pen_apply(l[i], c[i], p->repetition_penalty, p->frequency_penalty, p->presence_penalty);
  for (int j = 0; j < p->n_bias; j++) out[p->bias_token[j]] = lnb_pen_bias(out[p->bias_token[j]], p->bias[j]);
  free(c);
}
/* rows x V logits, row r with parameters p[r], history hist[r][hist_len] and p_next[r] -> out[rows][V] */
void orc_penalize_rows(const float* l, int rows, int V, const lnb_penalties* p, const int32_t* hist, int hist_len, const int32_t* p_next,
                       float* out) {
  for (int r = 0; r < rows; r++)
    orc_penalize_row(l + (size_t)r * V, V, p + r, hist + (size_t)r * hist_len, p_next[r], out + (size_t)r * V);
}

/* rows x V logits -> rows tokens, parameters per row */
void orc_sample_rows(const float* l, int rows, int V, const float* T, const int32_t* K, const float* P, const uint64_t* seed,
                     const int64_t* p_next, int32_t* out) {
  for (int r = 0; r < rows; r++) out[r] = orc_sample_row(l + (size_t)r * V, V, T[r], K[r], P[r], seed[r], p_next[r]);
}

/* orc_generate (generateTokensInternal, inference.go:173-254) with the sampler in place of the argmax: the token for
 * position cur is drawn with p_next = cur */
int orc_generate_sampled(const orc_model* m, int vocab, const int32_t* prompt, int n_prompt, int seq_len, const int32_t* stop_ids,
                         int n_stop, float T, int32_t K, float P, uint64_t seed, int32_t* out) {
  if (n_prompt >= seq_len) return -1;
  orc_session* s = orc_session_new(m, seq_len);
  int32_t* tokens = (int32_t*)malloc((size_t)seq_len * 4);
  for (int i = 0; i < seq_len; i++) tokens[i] = -1;
  for (int i = 0; i < n_prompt; i++) tokens[i] = prompt[i];
  float* logits = (float*)malloc((size_t)vocab * sizeof(float));
  int prev = 0, n_out = 0;
  for (int cur = n_prompt; cur < seq_len; cur++) {
    if (orc_forward(m, s, tokens + prev, cur - prev, prev, logits, 0, NULL) != 0) { n_out = -1; break; }
    int32_t next = orc_sample_row(logits, vocab, T, K, P, seed, cur);
    if (tokens[cur] != -1) next = tokens[cur];
    tokens[cur] = next;
    out[n_out++] = next;
    prev = cur;
    int eos = 0;
    for (int i = 0; i < n_stop; i++) eos |= (stop_ids[i] == next);
    if (eos) break;
    if (cur + 1 == seq_len) break;
  }
  free(tokens); free(logits);
  orc_session_free(s);
  return n_out;
}

/* orc_generate_sampled with the penalties in front of the sampler (greedy at T = 0): the token for position cur is drawn
 * from orc_penalize_row of the logits with the tokens fed at [0, cur) (pen NULL: orc_generate_sampled) */
int orc_generate_processed(const orc_model* m, int vocab, const int32_t* prompt, int n_prompt, int seq_len, const int32_t* stop_ids,
                           int n_stop, float T, int32_t K, float P, uint64_t seed, const lnb_penalties* pen, int32_t* out) {
  if (n_prompt >= seq_len) return -1;
  orc_session* s = orc_session_new(m, seq_len);
  int32_t* tokens = (int32_t*)malloc((size_t)seq_len * 4);
  for (int i = 0; i < seq_len; i++) tokens[i] = -1;
  for (int i = 0; i < n_prompt; i++) tokens[i] = prompt[i];
  float* logits = (float*)malloc((size_t)vocab * sizeof(float));
  float* proc = (float*)malloc((size_t)vocab * sizeof(float));
  int prev = 0, n_out = 0;
  for (int cur = n_prompt; cur < seq_len; cur++) {
    if (orc_forward(m, s, tokens + prev, cur - prev, prev, logits, 0, NULL) != 0) { n_out = -1; break; }
    if (pen) orc_penalize_row(logits, vocab, pen, tokens, cur, proc);
    int32_t next = orc_sample_row(pen ? proc : logits, vocab, T, K, P, seed, cur);
    if (tokens[cur] != -1) next = tokens[cur];
    tokens[cur] = next;
    out[n_out++] = next;
    prev = cur;
    int eos = 0;
    for (int i = 0; i < n_stop; i++) eos |= (stop_ids[i] == next);
    if (eos) break;
    if (cur + 1 == seq_len) break;
  }
  free(tokens); free(logits); free(proc);
  orc_session_free(s);
  return n_out;
}
