/* Sequential C statement of the seeded sampler (TEST INFRASTRUCTURE, NOT PRODUCT CODE; DESIGN.md §9b).
 *
 * The reference (inference.go:207-216) only has the greedy ml.Argmax, so sampling is an extension; this file states its
 * contract in the plainest form -- a full sort for the rank order, sequential integer sums -- for the tests to hold the
 * sampler kernel (csrc/sample.cuh) against.  The floating-point steps come from csrc/sample_det.h, the header the kernel
 * compiles too.  orc_generate_sampled drives the CPU oracle's forward (oracle/lnb_oracle.h) like orc_generate, with the
 * sampler in place of the argmax. */
#include <math.h>
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

/* ---- beam search (DESIGN.md §9f), written from the contract: the selection, the pool and the end rules in plain C ------ */
#include <math.h>

typedef struct {
  double score;
  int32_t beam, rank, token;
  double lp;
} orc_beam_cand;

/* score descending, -inf after every finite score, NaN last; then beam ascending; then rank ascending */
static int beam_score_cmp(double a, double b) {
  const int na = isnan(a), nb = isnan(b);
  if (na || nb) return na - nb;
  return a > b ? -1 : a < b ? 1 : 0;
}
static int beam_cand_cmp(const void* pa, const void* pb) {
  const orc_beam_cand *a = (const orc_beam_cand*)pa, *b = (const orc_beam_cand*)pb;
  const int c = beam_score_cmp(a->score, b->score);
  if (c) return c;
  if (a->beam != b->beam) return a->beam < b->beam ? -1 : 1;
  return a->rank < b->rank ? -1 : a->rank > b->rank ? 1 : 0;
}
static int beam_is_stop(int32_t t, const int32_t* stop, int n_stop) {
  for (int i = 0; i < n_stop; i++)
    if (stop[i] == t) return 1;
  return 0;
}
/* sorts c[n] in place; new_idx[*n_new] / fin_idx[*n_fin]: positions in the sorted list of the new beams and the finished */
static void beam_select(orc_beam_cand* c, int n, int B, const int32_t* stop, int n_stop, int32_t* new_idx, int* n_new,
                        int32_t* fin_idx, int* n_fin) {
  qsort(c, (size_t)n, sizeof(orc_beam_cand), beam_cand_cmp);
  *n_new = *n_fin = 0;
  for (int i = 0; i < n && *n_new < B; i++) {
    if (beam_is_stop(c[i].token, stop, n_stop)) {
      if (i < B) fin_idx[(*n_fin)++] = i;
    } else {
      new_idx[(*n_new)++] = i;
    }
  }
}
/* the selection alone on a candidate table (for the tests): the sorted table back in score/beam/rank/token, and the indices */
void orc_beam_select(double* score, int32_t* beam, int32_t* rank, int32_t* token, int n, int B, const int32_t* stop, int n_stop,
                     int32_t* new_idx, int32_t* n_new, int32_t* fin_idx, int32_t* n_fin) {
  orc_beam_cand* c = (orc_beam_cand*)malloc((size_t)(n > 0 ? n : 1) * sizeof(orc_beam_cand));
  for (int i = 0; i < n; i++) { c[i].score = score[i]; c[i].beam = beam[i]; c[i].rank = rank[i]; c[i].token = token[i]; c[i].lp = 0; }
  int nn, nf;
  beam_select(c, n, B, stop, n_stop, new_idx, &nn, fin_idx, &nf);
  for (int i = 0; i < n; i++) { score[i] = c[i].score; beam[i] = c[i].beam; rank[i] = c[i].rank; token[i] = c[i].token; }
  *n_new = nn;
  *n_fin = nf;
  free(c);
}

typedef struct {
  int32_t* tok;   /* [seq_len] */
  double* lp;     /* [seq_len] */
  int len;
  double s, h;
  int state;      /* 1: EOS, 2: SeqLen */
  int64_t ins;
} orc_beam_hyp;

/* a worse than b in the pool: lower h (NaN lowest), on equal h the later insertion */
static int beam_hyp_worse(const orc_beam_hyp* a, const orc_beam_hyp* b) {
  const int c = beam_score_cmp(a->h, b->h);
  if (c) return c > 0;
  return a->ins > b->ins;
}
typedef struct {
  int B, n, seq_len;
  int64_t n_ins;
  orc_beam_hyp* e;
} orc_beam_pool;
static int beam_pool_worst(const orc_beam_pool* p) {
  int w = 0;
  for (int j = 1; j < p->n; j++)
    if (beam_hyp_worse(&p->e[j], &p->e[w])) w = j;
  return w;
}
static void beam_pool_add(orc_beam_pool* p, const int32_t* tok, const double* lp, int len, double s, double h, int state) {
  orc_beam_hyp* slot;
  const int64_t ins = p->n_ins++;
  if (p->n < p->B) {
    slot = &p->e[p->n++];
  } else {
    const int w = beam_pool_worst(p);
    if (beam_score_cmp(h, p->e[w].h) >= 0) return;   /* not strictly better: the earlier insertion keeps its place */
    slot = &p->e[w];
  }
  memcpy(slot->tok, tok, (size_t)len * 4);
  memcpy(slot->lp, lp, (size_t)len * 8);
  slot->len = len; slot->s = s; slot->h = h; slot->state = state; slot->ins = ins;
}
/* the pool rule alone (for the tests): hypotheses with normalised scores h[n] inserted in order into a pool of B; kept[]
 * gets the indices the pool ends with, best first (ties: insertion order); returns how many, -1 for B outside [1, 8] */
int orc_beam_pool_run(const double* h, int n, int B, int32_t* kept) {
  if (B < 1 || B > 8) return -1;
  orc_beam_pool p = {B, 0, 1, 0, (orc_beam_hyp*)calloc((size_t)B, sizeof(orc_beam_hyp))};
  int32_t dummy_t = 0;
  double dummy_l = 0;
  for (int j = 0; j < B; j++) { p.e[j].tok = (int32_t*)malloc(4); p.e[j].lp = (double*)malloc(8); }
  for (int i = 0; i < n; i++) beam_pool_add(&p, &dummy_t, &dummy_l, 0, 0.0, h[i], 1);
  int m = 0;
  for (int used[8] = {0}; m < p.n; m++) {   /* selection sort: best first */
    int b = -1;
    for (int j = 0; j < p.n; j++)
      if (!used[j] && (b < 0 || beam_hyp_worse(&p.e[b], &p.e[j]))) b = j;
    used[b] = 1;
    kept[m] = (int32_t)p.e[b].ins;
  }
  for (int j = 0; j < B; j++) { free(p.e[j].tok); free(p.e[j].lp); }
  free(p.e);
  return m;
}

/* what the search reads and moves: the model side (an oracle model below, a table in the tests) */
typedef struct {
  void* ctx;
  /* step k: the rows after the prompt (k == 0, beam 0 only, n == 1) or after beam b was fed last[b] at position L + k - 1;
   * writes beam b's top tokens and logprobs to top_tok[b * 20 ..], top_lp[b * 20 ..], their count to n_top[b] */
  int (*step)(void* ctx, int k, int n, const int32_t* last, int32_t* top_tok, double* top_lp, int32_t* n_top);
  /* beams dst[i] take rows [pos0, pos1) of beam src[i], read as a snapshot */
  int (*reorder)(void* ctx, int n, const int32_t* src, const int32_t* dst, int pos0, int pos1);
} orc_beam_io;

/* The search of DESIGN.md §9f.  Results (best first) to out_tok[h * seq_len ..], out_lp[h * seq_len ..], out_len[h],
 * out_s[h], out_h[h], out_state[h] (1 EOS, 2 SeqLen); moves[] (or NULL) counts the copies whose parent differs from the
 * beam; returns the number of hypotheses, -1 on an error of io */
int orc_beam_search_io(const orc_beam_io* io, int n_prompt, int seq_len, const int32_t* stop, int n_stop, int B, double alpha,
                       int early, int32_t* out_tok, double* out_lp, int32_t* out_len, double* out_s, double* out_h, int32_t* out_state) {
  if (B < 1 || B > 8 || n_prompt < 1 || n_prompt >= seq_len) return -1;
  const int L = n_prompt, TOPW = 20;
  orc_beam_pool pool = {B, 0, seq_len, 0, (orc_beam_hyp*)calloc((size_t)B, sizeof(orc_beam_hyp))};
  for (int j = 0; j < B; j++) { pool.e[j].tok = (int32_t*)malloc((size_t)seq_len * 4); pool.e[j].lp = (double*)malloc((size_t)seq_len * 8); }
  /* live beams, and the next step's beams */
  int32_t *tok = (int32_t*)malloc((size_t)B * seq_len * 4), *tok2 = (int32_t*)malloc((size_t)B * seq_len * 4);
  double *lp = (double*)malloc((size_t)B * seq_len * 8), *lp2 = (double*)malloc((size_t)B * seq_len * 8);
  double s[8], s2[8];
  int n_live = 1, len = 0, rc = 0;
  s[0] = 0.0;
  int32_t top_tok[8 * 20], n_top[8], last[8], parent[8], new_idx[8 * 20], fin_idx[8 * 20];
  double top_lp[8 * 20];
  orc_beam_cand* c = (orc_beam_cand*)malloc((size_t)8 * TOPW * sizeof(orc_beam_cand));
  for (int k = 0; k < seq_len - L; k++) {
    for (int b = 0; b < n_live; b++) last[b] = len ? tok[b * seq_len + len - 1] : -1;
    if (io->step(io->ctx, k, n_live, last, top_tok, top_lp, n_top)) { rc = -1; break; }
    int nc = 0;
    for (int b = 0; b < n_live; b++)
      for (int j = 0; j < n_top[b]; j++) {
        c[nc].score = s[b] + top_lp[b * TOPW + j];
        c[nc].beam = b; c[nc].rank = j; c[nc].token = top_tok[b * TOPW + j]; c[nc].lp = top_lp[b * TOPW + j];
        nc++;
      }
    int nn, nf;
    beam_select(c, nc, B, stop, n_stop, new_idx, &nn, fin_idx, &nf);
    for (int f = 0; f < nf; f++) {   /* finished: the parent's tokens and this one */
      const orc_beam_cand* x = &c[fin_idx[f]];
      int32_t* t = tok + (size_t)x->beam * seq_len;
      double* l = lp + (size_t)x->beam * seq_len;
      const int32_t keep_t = t[len];
      const double keep_l = l[len];
      t[len] = x->token; l[len] = x->lp;
      beam_pool_add(&pool, t, l, len + 1, x->score, x->score / pow((double)(len + 1), alpha), 1);
      t[len] = keep_t; l[len] = keep_l;
    }
    if (nn < B) break;   /* fewer than B new beams: the search ends with the pool it has */
    for (int i = 0; i < B; i++) {
      const orc_beam_cand* x = &c[new_idx[i]];
      parent[i] = x->beam;
      memcpy(tok2 + (size_t)i * seq_len, tok + (size_t)x->beam * seq_len, (size_t)len * 4);
      memcpy(lp2 + (size_t)i * seq_len, lp + (size_t)x->beam * seq_len, (size_t)len * 8);
      tok2[(size_t)i * seq_len + len] = x->token;
      lp2[(size_t)i * seq_len + len] = x->lp;
      s2[i] = x->score;
    }
    { int32_t* t = tok; tok = tok2; tok2 = t; double* l = lp; lp = lp2; lp2 = l; }
    memcpy(s, s2, sizeof(s));
    n_live = B;
    len++;
    if (L + k == seq_len - 1) {   /* the new tokens sit at the last position: every live beam finishes, in beam order */
      for (int b = 0; b < B; b++)
        beam_pool_add(&pool, tok + (size_t)b * seq_len, lp + (size_t)b * seq_len, len, s[b], s[b] / pow((double)len, alpha), 2);
      break;
    }
    if (pool.n == B) {
      double hb = s[0] / pow((double)len, alpha);   /* the best live h */
      for (int b = 1; b < B; b++) {
        const double h = s[b] / pow((double)len, alpha);
        if (beam_score_cmp(h, hb) < 0) hb = h;
      }
      if (early || beam_score_cmp(hb, pool.e[beam_pool_worst(&pool)].h) >= 0) break;
    }
    int32_t src[8], dst[8];
    int nm = 0;
    for (int i = 0; i < B; i++)
      if (parent[i] != i) { src[nm] = parent[i]; dst[nm] = i; nm++; }
    if (nm && io->reorder(io->ctx, nm, src, dst, k == 0 ? 0 : L, L + k)) { rc = -1; break; }
  }
  int n_out = 0;
  if (rc == 0) {
    int used[8] = {0};
    for (; n_out < pool.n; n_out++) {   /* best first, ties in insertion order */
      int b = -1;
      for (int j = 0; j < pool.n; j++)
        if (!used[j] && (b < 0 || beam_hyp_worse(&pool.e[b], &pool.e[j]))) b = j;
      used[b] = 1;
      const orc_beam_hyp* x = &pool.e[b];
      memcpy(out_tok + (size_t)n_out * seq_len, x->tok, (size_t)x->len * 4);
      memcpy(out_lp + (size_t)n_out * seq_len, x->lp, (size_t)x->len * 8);
      out_len[n_out] = x->len; out_s[n_out] = x->s; out_h[n_out] = x->h; out_state[n_out] = x->state;
    }
  }
  for (int j = 0; j < B; j++) { free(pool.e[j].tok); free(pool.e[j].lp); }
  free(pool.e); free(tok); free(tok2); free(lp); free(lp2); free(c);
  return rc ? -1 : n_out;
}

/* the oracle model side: B sessions, orc_forward per beam at S = 1, orc_logprob_row(top_n = min(2B, V)) of each row;
 * reorder by memcpy of the caches through a snapshot of every source */
typedef struct {
  const orc_model* m;
  int vocab, B, seq_len, n_layers, kv_row;   /* kv_row: elements per position of one cache */
  const int32_t* prompt;
  int n_prompt;
  orc_session* s[8];
  float* logits;
  uint16_t* snap;
  int64_t* n_moves;
} orc_beam_oracle;

static int beam_oracle_step(void* ctx, int k, int n, const int32_t* last, int32_t* top_tok, double* top_lp, int32_t* n_top) {
  orc_beam_oracle* o = (orc_beam_oracle*)ctx;
  const int top_n = 2 * o->B < o->vocab ? 2 * o->B : o->vocab;
  lnb_logprob rec;
  for (int b = 0; b < n; b++) {
    const int rc = k == 0 ? orc_forward(o->m, o->s[0], o->prompt, o->n_prompt, 0, o->logits, 0, NULL)
                          : orc_forward(o->m, o->s[b], last + b, 1, o->n_prompt + k - 1, o->logits, 0, NULL);
    if (rc != 0) return -1;
    orc_logprob_row(o->logits, o->vocab, 0, top_n, &rec);
    n_top[b] = rec.n_top;
    for (int j = 0; j < rec.n_top; j++) { top_tok[b * 20 + j] = rec.top_token[j]; top_lp[b * 20 + j] = rec.top_logprob[j]; }
  }
  return 0;
}
static int beam_oracle_reorder(void* ctx, int n, const int32_t* src, const int32_t* dst, int pos0, int pos1) {
  orc_beam_oracle* o = (orc_beam_oracle*)ctx;
  const size_t off = (size_t)pos0 * o->kv_row, cnt = (size_t)(pos1 - pos0) * o->kv_row;
  for (int l = 0; l < o->n_layers; l++)
    for (int kv = 0; kv < 2; kv++) {
      for (int i = 0; i < n; i++) {   /* snapshot of every source first ... */
        const uint16_t* c = kv ? orc_session_cache_v(o->s[src[i]], l) : orc_session_cache_k(o->s[src[i]], l);
        memcpy(o->snap + (size_t)i * cnt, c + off, cnt * 2);
      }
      for (int i = 0; i < n; i++) {   /* ... then the destinations */
        uint16_t* c = kv ? orc_session_cache_v(o->s[dst[i]], l) : orc_session_cache_k(o->s[dst[i]], l);
        memcpy(c + off, o->snap + (size_t)i * cnt, cnt * 2);
      }
    }
  if (o->n_moves) (*o->n_moves)++;
  return 0;
}

/* beam search on the oracle model (n_layers and kv_row = n_kv_heads * head_dim describe its caches); n_moves (or NULL)
 * counts the reorders */
int orc_beam_search(const orc_model* m, int vocab, int n_layers, int kv_row, const int32_t* prompt, int n_prompt, int seq_len,
                    const int32_t* stop, int n_stop, int B, double alpha, int early, int32_t* out_tok, double* out_lp,
                    int32_t* out_len, double* out_s, double* out_h, int32_t* out_state, int64_t* n_moves) {
  if (B < 1 || B > 8) return -1;
  orc_beam_oracle o = {m, vocab, B, seq_len, n_layers, kv_row, prompt, n_prompt, {0}, NULL, NULL, n_moves};
  for (int b = 0; b < B; b++) o.s[b] = orc_session_new(m, seq_len);
  o.logits = (float*)malloc((size_t)vocab * n_prompt * sizeof(float));
  o.snap = (uint16_t*)malloc((size_t)B * seq_len * kv_row * 2);
  if (n_moves) *n_moves = 0;
  const orc_beam_io io = {&o, beam_oracle_step, beam_oracle_reorder};
  const int n = orc_beam_search_io(&io, n_prompt, seq_len, stop, n_stop, B, alpha, early, out_tok, out_lp, out_len, out_s, out_h,
                                   out_state);
  for (int b = 0; b < B; b++) orc_session_free(o.s[b]);
  free(o.logits); free(o.snap);
  return n;
}

/* ---- grammars (DESIGN.md §9g), written from the contract of include/lnb.h: brute-force masks and the state history ---- */
/* a grammar's tables: trans[Q][256] (-1: ⊥), accept[Q], token t's bytes bytes[off[t] .. off[t+1]), the stop set */
typedef struct {
  const int32_t* trans;
  const uint8_t* accept;
  int Q;
  const uint8_t* bytes;
  const int64_t* off;
  int V;
  const int32_t* stop;
  int n_stop;
} orc_grammar;

static int grm_is_stop(const orc_grammar* g, int32_t t) {
  for (int i = 0; i < g->n_stop; i++)
    if (g->stop[i] == t) return 1;
  return 0;
}
/* δ*(q, b(t)) */
static int grm_walk(const orc_grammar* g, int q, int32_t t) {
  for (int64_t i = g->off[t]; i < g->off[t + 1] && q >= 0; i++) q = g->trans[(size_t)q * 256 + g->bytes[i]];
  return q;
}
static int grm_text_allowed(const orc_grammar* g, int q, int32_t t) {
  return q >= 0 && !grm_is_stop(g, t) && g->off[t + 1] > g->off[t] && grm_walk(g, q, t) >= 0;
}
/* the state after feeding t in q: δ*(q, b(t)) if t is an allowed text token in q, else ⊥ */
static int grm_next(const orc_grammar* g, int q, int32_t t) {
  return (t >= 0 && t < g->V && grm_text_allowed(g, q, t)) ? grm_walk(g, q, t) : -1;
}
/* mask(q) as a 0/1 byte per token (q = -1: ⊥) */
static void grm_mask(const orc_grammar* g, int q, uint8_t* m) {
  int any = 0;
  for (int t = 0; t < g->V; t++) {
    m[t] = q >= 0 && (grm_is_stop(g, t) ? g->accept[q] != 0 : grm_text_allowed(g, q, t));
    any |= m[t];
  }
  if (!any)
    for (int t = 0; t < g->V; t++) m[t] = (uint8_t)grm_is_stop(g, t);
}

/* every state's mask, rows 0..Q-1, then ⊥'s as row Q, as u32 words [Q + 1][ceil(V / 32)] (bit t & 31 of word t >> 5);
 * returns the number of states whose mask is Z */
int orc_grammar_masks(const int32_t* trans, const uint8_t* accept, int Q, const uint8_t* bytes, const int64_t* off, int V,
                      const int32_t* stop, int n_stop, uint32_t* out) {
  const orc_grammar g = {trans, accept, Q, bytes, off, V, stop, n_stop};
  const int W = (V + 31) / 32;
  int stuck = 0;
#pragma omp parallel for reduction(+ : stuck) schedule(dynamic, 1)
  for (int q = -1; q < Q; q++) {
    uint8_t* m = (uint8_t*)malloc((size_t)V);
    grm_mask(&g, q, m);
    uint32_t* row = out + (size_t)(q < 0 ? Q : q) * W;
    memset(row, 0, (size_t)W * 4);
    int text = 0;
    for (int t = 0; t < V; t++) {
      if (m[t]) row[t >> 5] |= 1u << (t & 31);
      text |= m[t] && !grm_is_stop(&g, t);
    }
    if (q >= 0 && !text && !accept[q]) stuck++;
    free(m);
  }
  return stuck;
}

/* the state history of tokens[0 .. n) fed at positions 0 .. n-1 with the grammar starting at first_pos: hist[p] for
 * p in [0, n], -1 (⊥) below first_pos */
void orc_grammar_history(const int32_t* trans, const uint8_t* accept, int Q, const uint8_t* bytes, const int64_t* off, int V,
                         const int32_t* stop, int n_stop, const int32_t* tokens, int n, int first_pos, int32_t* hist) {
  const orc_grammar g = {trans, accept, Q, bytes, off, V, stop, n_stop};
  for (int p = 0; p <= n; p++) hist[p] = -1;
  if (first_pos > n) return;
  hist[first_pos] = 0;
  for (int p = first_pos; p < n; p++) hist[p + 1] = grm_next(&g, hist[p], tokens[p]);
}

/* orc_generate_processed with the grammar: the row that emits position p >= first_pos keeps the logits of mask(g[p]) only,
 * between the penalties and the sampler */
int orc_generate_constrained(const orc_model* m, int vocab, const int32_t* prompt, int n_prompt, int seq_len, const int32_t* stop_ids,
                             int n_stop, float T, int32_t K, float P, uint64_t seed, const lnb_penalties* pen,
                             const int32_t* trans, const uint8_t* accept, int Q, const uint8_t* bytes, const int64_t* off,
                             const int32_t* grammar_stop, int n_grammar_stop, int first_pos, int32_t* out) {
  if (n_prompt >= seq_len) return -1;
  const orc_grammar g = {trans, accept, Q, bytes, off, vocab, grammar_stop, n_grammar_stop};
  orc_session* s = orc_session_new(m, seq_len);
  int32_t* tokens = (int32_t*)malloc((size_t)seq_len * 4);
  int32_t* hist = (int32_t*)malloc((size_t)(seq_len + 1) * 4);
  for (int i = 0; i < seq_len; i++) tokens[i] = -1;
  for (int i = 0; i < n_prompt; i++) tokens[i] = prompt[i];
  for (int p = 0; p <= seq_len; p++) hist[p] = -1;
  if (first_pos <= seq_len) hist[first_pos] = 0;
  float* logits = (float*)malloc((size_t)vocab * sizeof(float));
  float* proc = (float*)malloc((size_t)vocab * sizeof(float));
  uint8_t* mask = (uint8_t*)malloc((size_t)vocab);
  int prev = 0, n_out = 0, walked = first_pos;   /* hist[first_pos .. walked] are known */
  for (int cur = n_prompt; cur < seq_len; cur++) {
    if (orc_forward(m, s, tokens + prev, cur - prev, prev, logits, 0, NULL) != 0) { n_out = -1; break; }
    if (pen) orc_penalize_row(logits, vocab, pen, tokens, cur, proc);
    else memcpy(proc, logits, (size_t)vocab * sizeof(float));
    if (cur >= first_pos) {
      for (; walked < cur; walked++) hist[walked + 1] = grm_next(&g, hist[walked], tokens[walked]);
      grm_mask(&g, hist[cur], mask);
      for (int t = 0; t < vocab; t++)
        if (!mask[t]) proc[t] = -INFINITY;
    }
    const int32_t next = orc_sample_row(proc, vocab, T, K, P, seed, cur);
    tokens[cur] = next;
    out[n_out++] = next;
    prev = cur;
    int eos = 0;
    for (int i = 0; i < n_stop; i++) eos |= (stop_ids[i] == next);
    if (eos) break;
    if (cur + 1 == seq_len) break;
  }
  free(tokens); free(hist); free(logits); free(proc); free(mask);
  orc_session_free(s);
  return n_out;
}

/* ---- MXFP8 weights (DESIGN.md §9h; the device form is csrc/mxfp8.cuh) ------------------------------------------------
 * w: a row-major bf16 matrix [rows][cols]; codes [rows][cols], scales [rows][ceil(cols / 32)].  Each run of 32 columns of a
 * row (the last one shorter) is a block: X = floor(log2(amax)) - 8 clamped to [-117, 119] (-117 for a zero block), scale
 * byte X + 127; code = E4M3 of w * 2^-X, round to nearest even, magnitudes of 448 and above saturated to 448 (0x7E).  The
 * scaled value is formed exactly in double.  Returns -1, or row * cols + col of the first non-finite weight (nothing is
 * written then). */
static uint8_t e4m3_rne_sat(double v) {
  const uint8_t sign = signbit(v) ? 0x80 : 0;
  const double a = fabs(v);
  if (a >= 448.0) return sign | 0x7E;
  if (a < 0x1p-6) return sign | (uint8_t)rint(a * 0x1p9);   /* subnormal quantum 2^-9; 8 quanta carry into 2^-6 = 0x08 */
  int e;
  frexp(a, &e);                                              /* a = f * 2^e, f in [0.5, 1): binade 2^(e-1) */
  const double r = rint(ldexp(a, 3 - (e - 1)));              /* 8..16 eighths of the binade */
  return sign | (uint8_t)((((e - 1) + 7) << 3) + (int)r - 8); /* r == 16 carries into the next binade */
}
int64_t orc_mxfp8_quantize(const uint16_t* w, int rows, int cols, uint8_t* codes, uint8_t* scales) {
  for (int64_t i = 0; i < (int64_t)rows * cols; i++)
    if ((w[i] & 0x7f80) == 0x7f80) return i;
  const int nb = (cols + 31) / 32;
  for (int r = 0; r < rows; r++)
    for (int b = 0; b < nb; b++) {
      const int c0 = b * 32, c1 = c0 + 32 < cols ? c0 + 32 : cols;
      uint16_t amax = 0;
      for (int c = c0; c < c1; c++) {
        const uint16_t mag = w[(int64_t)r * cols + c] & 0x7fff;
        if (mag > amax) amax = mag;
      }
      const int E = amax >> 7;
      int X = E == 0 ? -117 : E - 127 - 8;
      if (X < -117) X = -117;
      if (X > 119) X = 119;
      scales[(int64_t)r * nb + b] = (uint8_t)(X + 127);
      for (int c = c0; c < c1; c++) {
        const uint32_t bits = (uint32_t)w[(int64_t)r * cols + c] << 16;
        float f;
        memcpy(&f, &bits, 4);
        codes[(int64_t)r * cols + c] = e4m3_rne_sat(ldexp((double)f, -X));
      }
    }
  return -1;
}
/* e4m3(code) * 2^X as bf16 bits (exact: the value is zero or a normal number of at most 4 significant bits, so the f32
 * product of the code's value and 2^X, X in [-117, 119], is exact too) */
void orc_mxfp8_dequantize(const uint8_t* codes, const uint8_t* scales, int rows, int cols, uint16_t* out) {
  float val[256];
  for (int q = 0; q < 256; q++) {
    const int e = (q >> 3) & 15, mnt = q & 7;
    const double v = (q & 0x7f) == 0x7f ? NAN : e == 0 ? ldexp((double)mnt, -9) : ldexp(8.0 + mnt, e - 7 - 3);
    val[q] = (float)((q & 0x80) ? -v : v);
  }
  const int nb = (cols + 31) / 32;
  for (int r = 0; r < rows; r++)
    for (int c = 0; c < cols; c++) {
      const int X = (int)scales[(int64_t)r * nb + c / 32] - 127;
      const float f = val[codes[(int64_t)r * cols + c]] * ldexpf(1.0f, X);
      uint32_t bits;
      memcpy(&bits, &f, 4);
      out[(int64_t)r * cols + c] = (uint16_t)(bits >> 16);
    }
}

/* MXFP8 KV cache (DESIGN.md §9j; the device form is csrc/kvcache.cuh): rows [n][n_kv * head_dim] bf16 -> codes
 * [n][n_kv * head_dim], scales [n][n_kv][ceil(head_dim / 32)] and (deq != NULL) e4m3(code) * 2^X as bf16 bits.  The rule of
 * orc_mxfp8_quantize on the matrix of head rows [n * n_kv][head_dim], except that K and V rows cannot be refused: the block
 * maximum is taken over the finite elements, a NaN element stores the NaN code 0x7F (decoded 0x7FC0) and +-inf saturates
 * to +-448 (0x7E with the sign). */
void orc_kv_mxfp8_quantize(const uint16_t* rows, int n, int head_dim, int n_kv, uint8_t* codes, uint8_t* scales, uint16_t* deq) {
  const int64_t ne = (int64_t)n * n_kv * head_dim;
  if (ne <= 0) return;
  uint16_t* fin = (uint16_t*)malloc((size_t)ne * 2);
  for (int64_t i = 0; i < ne; i++) fin[i] = (rows[i] & 0x7f80) == 0x7f80 ? (uint16_t)(rows[i] & 0x8000) : rows[i];
  orc_mxfp8_quantize(fin, n * n_kv, head_dim, codes, scales);
  free(fin);
  for (int64_t i = 0; i < ne; i++)
    if ((rows[i] & 0x7f80) == 0x7f80) codes[i] = (rows[i] & 0x7f) ? 0x7F : (uint8_t)(((rows[i] >> 8) & 0x80) | 0x7E);
  if (deq) orc_mxfp8_dequantize(codes, scales, n * n_kv, head_dim, deq);
}

/* MXFP4 linear weights (DESIGN.md §9i): the MXFP8 blocks, one E2M1 code per weight, packed two a byte with the even
 * column in the low nibble: codes [rows][cols / 2], scales [rows][ceil(cols / 32)].  X = e - 2 if the 7-bit mantissa field
 * f of the bf16 block maximum is <= 64, else e - 1 (e its unbiased exponent), clamped to [-125, 125]; -125 for a zero or
 * subnormal maximum.  code = sign bit | |w| * 2^-X rounded to the nearest of {0, 0.5, 1, 1.5, 2, 3, 4, 6}, ties to the even
 * mantissa bit (index), saturated at 6.  Returns the index of the first non-finite weight, or -1. */
int64_t orc_mxfp4_quantize(const uint16_t* w, int rows, int cols, uint8_t* codes, uint8_t* scales) {
  static const double grid[8] = {0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0};
  for (int64_t i = 0; i < (int64_t)rows * cols; i++)
    if ((w[i] & 0x7f80) == 0x7f80) return i;
  const int nb = (cols + 31) / 32;
  memset(codes, 0, (size_t)rows * (cols / 2));
  for (int r = 0; r < rows; r++)
    for (int b = 0; b < nb; b++) {
      const int c0 = b * 32, c1 = c0 + 32 < cols ? c0 + 32 : cols;
      uint16_t amax = 0;
      for (int c = c0; c < c1; c++) {
        const uint16_t mag = w[(int64_t)r * cols + c] & 0x7fff;
        if (mag > amax) amax = mag;
      }
      const int E = amax >> 7;
      int X = E == 0 ? -125 : E - 127 - ((amax & 0x7f) <= 64 ? 2 : 1);
      if (X < -125) X = -125;
      if (X > 125) X = 125;
      scales[(int64_t)r * nb + b] = (uint8_t)(X + 127);
      for (int c = c0; c < c1; c++) {
        const uint16_t h = w[(int64_t)r * cols + c];
        const uint32_t bits = (uint32_t)(h & 0x7fff) << 16;
        float f;
        memcpy(&f, &bits, 4);
        const double q = ldexp((double)f, -X);
        int k = 0;   /* nearest grid point; on a tie the one with the even index */
        for (int j = 1; j < 8; j++) {
          const double d0 = q - grid[k], d1 = grid[j] - q;
          if (d1 < d0 || (d1 == d0 && (j & 1) == 0)) k = j;
        }
        const uint8_t code = (uint8_t)(((h >> 12) & 8) | k);
        codes[(int64_t)r * (cols / 2) + c / 2] |= (uint8_t)(code << (4 * (c & 1)));
      }
    }
  return -1;
}
/* e2m1(code) * 2^X as bf16 bits (exact: zero or a normal number of at most 2 significant bits inside the bf16 range) */
void orc_mxfp4_dequantize(const uint8_t* codes, const uint8_t* scales, int rows, int cols, uint16_t* out) {
  static const double grid[8] = {0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0};
  const int nb = (cols + 31) / 32;
  for (int r = 0; r < rows; r++)
    for (int c = 0; c < cols; c++) {
      const int code = (codes[(int64_t)r * (cols / 2) + c / 2] >> (4 * (c & 1))) & 15;
      const int X = (int)scales[(int64_t)r * nb + c / 32] - 127;
      const double v = ldexp(grid[code & 7], X);
      const float f = (float)((code & 8) ? -v : v);
      uint32_t bits;
      memcpy(&bits, &f, 4);
      out[(int64_t)r * cols + c] = (uint16_t)(bits >> 16);
    }
}
