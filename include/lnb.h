/*
 * lnb.h -- C-ABI of liblnb.so: the H100 (sm_90a) forward path that sits under the
 * Go API of adalkiran/llama-nuts-and-bolts.
 *
 * The reference has no FFI or plugin interface (it is pure Go, CPU only); the
 * drop-in boundary is its exported Go API, and this header is what a cgo shim in
 * src/ml and src/model binds (INTEGRATION.md shows the stubs).  Every entry point
 * cites the reference symbol (file:line, relative to the reference repo) whose
 * arithmetic it replaces.  Plain C types only; no pointer is retained past a call
 * (cgo pointer rule) -- weights are copied to HBM at upload.
 *
 * Error convention (reference: `(nil, error)` from every op, e.g.
 * src/ml/operations_impl.go:428-446): every function returns 0 on success or a
 * negative LNB_E* code; lnb_last_error() returns the thread-local message.
 *
 * Numeric contract (SURVEY.md Appendix A): bf16 storage, f32 accumulate,
 * f32 -> bf16 by TRUNCATION after every op (src/dtype/bfloat16.go:59-61), f64
 * softmax without max-subtraction, table SiLU, RoPE through f64 intermediates.
 * The accumulation ORDER of the long sums is selectable:
 *   LNB_ACC_STRICT  k = 0,1,2,... sequentially per output, exactly the reference's
 *                   order -> results are bit-identical to the Go CPU path.
 *   LNB_ACC_FAST    each output's sum is split into interleaved partial sums that
 *                   are combined in a fixed documented order (DESIGN.md) -> same
 *                   values up to fp32 summation order; faster (HBM-bound).
 */
#ifndef LNB_H
#define LNB_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LNB_VERSION 100

enum {
  LNB_OK = 0,
  LNB_EINVAL = -1,   /* bad argument / shape / dtype (reference: fmt.Errorf shape errors) */
  LNB_ECUDA = -2,    /* CUDA runtime failure (sticky on the handle) */
  LNB_ENCCL = -3,    /* NCCL failure */
  LNB_ESTATE = -4,   /* call order (e.g. forward before finalize) */
  LNB_ENOMEM = -5,
  LNB_ETIMEOUT = -6  /* a tensor-parallel peer did not deliver its all-reduce words in time (late / dead rank) */
};

enum { LNB_ACC_STRICT = 0, LNB_ACC_FAST = 1 };

const char* lnb_last_error(void);
int lnb_version(void);
/* number of visible CUDA devices, or a negative error */
int lnb_device_count(void);

/* ------------------------------------------------------------------------------------
 * Model-level API -- replaces model.NewLlamaTransformer / LlamaTransformer.Forward
 * ---------------------------------------------------------------------------------- */

/* mirrors model.ModelArgs (src/model/modelargs.go:10-64) plus the derived FFN width
 * (src/model/llamatransformer.go:569-577) */
typedef struct {
  int32_t dim, n_layers, n_heads, n_kv_heads, head_dim, ffn_dim, vocab_size, max_seq_len;
  float norm_eps;
  double rope_theta;
  int32_t use_scaled_rope;
} lnb_model_args;

typedef struct lnb_model lnb_model;     /* device-resident weights + tables of ONE rank */
typedef struct lnb_session lnb_session; /* model.InferenceContext: KV cache + activations */

/* Creates the device-side model of tensor-parallel rank `tp_rank` of `tp_size` on CUDA
 * device `device`.  tp_size==1: nccl_unique_id may be NULL.  tp_size>1: one process per
 * rank; nccl_unique_id is the 128-byte id from lnb_nccl_unique_id() of rank 0, sent by
 * the host (torch.distributed / Go) to every rank.
 * Shapes (LNB_EINVAL otherwise, before any device call): n_heads a multiple of n_kv_heads; head_dim a
 * multiple of 8 (every attention kernel reads a head's K/V row as 16-byte vectors); dim and each rank's
 * n_heads * head_dim and n_kv_heads * head_dim multiples of 32, its ffn_dim and vocab_size shares
 * multiples of 16.
 * Replaces: model.NewLlamaTransformer (src/model/llamatransformer.go:64-113). */
int lnb_model_create(const lnb_model_args* args, int device, int tp_rank, int tp_size,
                     const void* nccl_unique_id, lnb_model** out);
int lnb_nccl_unique_id(void* out128);
/* Host-only arithmetic (no CUDA call): the [row0:row0+rows, col0:col0+cols] window of checkpoint
 * tensor `name` that rank tp_rank of tp_size keeps (Megatron split: wq/wk/wv/w1/w3/output by rows,
 * wo/w2 by columns, norms and embeddings replicated; SURVEY.md 8e). */
int lnb_tp_shard_window(const lnb_model_args* args, const char* name, int tp_rank, int tp_size,
                        int64_t* row0, int64_t* col0, int64_t* rows, int64_t* cols);

/* Upload one checkpoint tensor by its reference name ("layers.7.attention.wq.weight",
 * "tok_embeddings.weight", ...; names and shapes: llamatransformer.go:84-105,191,202,
 * 273-282,580-586; getTensor shape check: src/model/loader.go:183-197).  `host` is the
 * FULL bf16 row-major [out,in] tensor exactly as it sits in the checkpoint mmap
 * (src/torch/types.go:51-56); the library copies (and, for tp_size>1, slices) it into
 * its HBM layout and keeps no reference to `host`. */
int lnb_model_upload_tensor(lnb_model* m, const char* name, const uint16_t* host, const int64_t* shape, int ndim);

/* ---- checkpoint files (SURVEY 8f-1) --------------------------------------------------------
 * Native reader / writer for PyTorch ".pth" archives (zip + pickle), host-only.
 * Replaces: torch.NewTorchModelReader / Load / persistentLoad (src/torch/torchmodelreader.go:21-145),
 * rebuild_tensor_v2 + TorchStorage.Load (src/torch/types.go:23-56), the unpickler (src/pickle/picklereader.go, pickledispatch.go)
 * and the read-only mmap (src/common/memorymapper_unix.go:21-45). */
typedef struct lnb_pth lnb_pth;
enum { LNB_PTH_BF16 = 0, LNB_PTH_F16 = 1, LNB_PTH_F32 = 2, LNB_PTH_F64 = 3, LNB_PTH_I8 = 4, LNB_PTH_U8 = 5,
       LNB_PTH_I16 = 6, LNB_PTH_I32 = 7, LNB_PTH_I64 = 8, LNB_PTH_BOOL = 9 };
/* maps the file, indexes the zip, unpickles the single *.pkl (torchmodelreader.go:39-66) */
int lnb_pth_open(const char* path, lnb_pth** out);
int lnb_pth_close(lnb_pth* f);
/* number of tensors in the top-level dict (pickle.PickleDict keys, torchmodelreader.go:57-63) */
int lnb_pth_tensor_count(const lnb_pth* f);
/* name / dtype / shape (<= 8 dims) / byte range inside the file of tensor `index` (dict order).
 * Returns 0, 1 when the tensor is not contiguous, or a negative error.  Any out pointer may be NULL. */
int lnb_pth_tensor_info(const lnb_pth* f, int index, const char** name, int* dtype, int* ndim, int64_t* shape,
                        int64_t* file_offset, int64_t* nbytes);
/* pointer into the read-only mapping (the reference's Tensor.RawData aliasing the mmap, types.go:51-56);
 * valid until lnb_pth_close */
const void* lnb_pth_tensor_data(const lnb_pth* f, int index);
/* model.LoadModelEx's tensor half (src/model/loader.go:22-41) fused with the by-name binding of
 * NewLlamaTransformer (llamatransformer.go:84-105): every tensor the architecture names goes from the page
 * cache to HBM (tp_size>1: only this rank's window); other entries are ignored.  lnb_model_finalize still
 * reports missing tensors. */
int lnb_model_load_pth(lnb_model* m, const char* path, int* n_uploaded);
/* loadModelArgsFromFile (src/model/modelargs.go:52-64) with the defaults of NewModelArgs (:29-44) and the
 * derived HeadDim / N_KVHeads / FFN width (llamatransformer.go:73-82,569-577).  vocab_size stays -1 when
 * params.json has none (the reference takes it from the tokenizer, loader.go:106-111). */
int lnb_model_args_from_params_json(const char* path, int max_seq_len, lnb_model_args* out);
/* writer: one storage per tensor at offset 0, pickle protocol 2 restricted to the opcodes the reference's
 * unpickler dispatches (src/pickle/pickledispatch.go:52-77) -- readable by torch.load and by the Go loader */
typedef struct lnb_pth_writer lnb_pth_writer;
int lnb_pth_writer_create(const char* path, lnb_pth_writer** out);
int lnb_pth_writer_add(lnb_pth_writer* w, const char* name, int dtype, const void* data, const int64_t* shape, int ndim);
/* writes data.pkl + the zip directory and frees the writer (also on failure) */
int lnb_pth_writer_finish(lnb_pth_writer* w);
/* the synthetic checkpoint of lnb_model_init_synthetic as a consolidated.00.pth (same bits, host-only) */
int lnb_pth_write_synthetic(const char* path, const lnb_model_args* args, uint64_t seed);

/* ---- tokenizer (SURVEY 8f-3) ------------------------------------------------------------------
 * tiktoken vocabulary + Llama-3 BPE, host-only.  Replaces tiktoken.Load (src/tiktoken/tiktokenreader.go:12-85),
 * model.NewVocabulary incl. its split regexp (src/model/vocabulary.go:23-50), InferenceEngine.TokenizeString /
 * bytePairMerge / Tokenize (src/inference/tokenize.go:27-193) and the byte concatenation under
 * TokenBatchToString (:239-258).  The console's emoji alias annotation (src/inference/emoji.go) is not built. */
typedef struct lnb_vocab lnb_vocab;
/* tokenizer.model: "<base64 token> <rank>" lines; the 256 special tokens are appended after the ranks */
int lnb_vocab_load(const char* tokenizer_model_path, lnb_vocab** out);
int lnb_vocab_destroy(lnb_vocab* v);
/* writes a stand-in tokenizer.model with n_mergeable ranks (256 bytes + unique 3-byte fillers that never merge) so that a
 * synthetic model directory passes checkModelArgs' VocabSize == vocabulary length (src/model/loader.go:98-120) */
int lnb_vocab_write_synthetic(const char* path, int n_mergeable);

/* len(Vocabulary.IdToToken) (vocabulary.go:27) */
int lnb_vocab_size(const lnb_vocab* v);
/* Vocabulary.TokenToId[token]; *id = -1 when absent.  `token` is raw bytes (pieces need not be valid UTF-8) */
int lnb_vocab_token_id(const lnb_vocab* v, const void* token, int token_len, int32_t* id);
/* Vocabulary.IdToToken[id]: pointer into the vocabulary, valid until lnb_vocab_destroy */
int lnb_vocab_token_bytes(const lnb_vocab* v, int32_t id, const void** bytes, int* len);
/* BeginOfSentenceId, EndOfSentenceId, PadId (-1) and the two StopTokenIds <|eom_id|>, <|eot_id|> (tiktokenreader.go:74-82) */
int lnb_vocab_special_ids(const lnb_vocab* v, int32_t* bos, int32_t* eos, int32_t* pad, int32_t* stop2);
/* Vocabulary.SplitRegexp.FindAllString (src/model/vocabulary.go:36, used at tokenize.go:180): byte offsets one past
 * each piece of `text`, by a hand-written matcher with Go/RE2 semantics (leftmost-first, ASCII \s, \p{L} / \p{N} of
 * Unicode 15.0, simple case folding in the contraction alternative) */
int lnb_split_pieces(const char* text, int64_t text_len, int64_t* ends, int cap, int* n_out);
/* InferenceEngine.TokenizeString (tokenize.go:175-193).  *n_out = tokens produced (also when cap is too small) */
int lnb_tokenize_string(const lnb_vocab* v, const char* text, int64_t text_len, int32_t* out, int cap, int* n_out);
/* InferenceEngine.Tokenize (tokenize.go:27-95): <|begin_of_text|>, every non-empty part wrapped in header tokens and
 * closed with <|eot_id|>, then the open assistant header */
int lnb_tokenize_prompt(const lnb_vocab* v, const char* const* headers, const char* const* contents, int n_parts,
                        int32_t* out, int cap, int* n_out);
/* bytes of the tokens up to the first PadId (TokenBatchToString :239-258 without the emoji annotation) */
int lnb_detokenize(const lnb_vocab* v, const int32_t* ids, int n, char* out, int64_t cap, int64_t* n_out);

/* Random-init every tensor directly in HBM with the synthetic generator of DESIGN.md
 * (no checkpoint exists in the build environment).  Same bits as oracle's
 * orc_synth_fill for the same seed. */
int lnb_model_init_synthetic(lnb_model* m, uint64_t seed);
/* host-side twin of the generator, for callers that want the same bytes in host memory */
int lnb_synth_fill_host(uint64_t seed, const char* name, float scale, float offset, int64_t n, uint16_t* out);
/* scale/offset used by lnb_model_init_synthetic for a tensor name */
int lnb_synth_spec(const lnb_model_args* args, const char* name, float* scale, float* offset);

/* Optional: override the tables the library builds itself at finalize.
 * cis: [rows][head_dim/2][2] f32 == model.precomputeFreqsCis output
 * (llamatransformer.go:694-751); silu_bf16: ml.TABLE_SILU truncated to bf16
 * (src/ml/activations.go:11-25,38). */
int lnb_model_set_rope_table(lnb_model* m, const float* cis, int rows);
int lnb_model_set_silu_table(lnb_model* m, const uint16_t* silu_bf16_65536);
/* read back the tables in use (tests compare them with the oracle's) */
int lnb_model_get_rope_table(lnb_model* m, float* cis_out, int rows);
int lnb_model_get_silu_table(lnb_model* m, uint16_t* out65536);

/* checks all 291 tensors are present, builds tables, makes the model immutable */
int lnb_model_finalize(lnb_model* m);
int lnb_model_destroy(lnb_model* m); /* hook for model.Model.Free (src/model/model.go:56) */
/* The packed copy the STRICT decode engine streams for w1|w3 of `layer` (layer -1: the LM head), built on first use
 * (DESIGN §4): data = [N/8 panels][12 * K] bytes, units = [N/8][k-tiles] unit bytes (0xFF = raw), src = the panel-major
 * bf16 it encodes [N/8][K/8][8][8]; any of them may be NULL.  info[5] = {kt, units, packed units, bytes the engine reads
 * per pass, N}.  Returns 1, or 0 when the engine streams bf16 (lnb_last_error says why).  The model must be finalized. */
int lnb_model_wpack_read(lnb_model* m, int layer, uint8_t* data, uint8_t* units, uint16_t* src, int64_t* info);

/* model.NewInferenceContext (src/model/inferencecontext.go:17-46): KV cache of seq_len rows
 * per layer, zero-filled.  max_rows = largest S a forward call may carry (>=1).
 * acc_mode = LNB_ACC_STRICT / LNB_ACC_FAST.
 * seq_len may be anything up to the model's max_seq_len (the RoPE table; LNB_EINVAL above it).  Sessions
 * whose seq_len the shared-memory attention kernel cannot hold (17 024 positions at head_dim 128) run every
 * row on the streamed attention kernels, which need head_dim <= 128 and n_heads / n_kv_heads <= 8.
 * LNB_ENOMEM when the caches and scratch do not fit the GPU (the message gives the bytes asked for);
 * nothing stays allocated then. */
int lnb_session_create(lnb_model* m, int seq_len, int max_rows, int acc_mode, lnb_session** out);
int lnb_session_destroy(lnb_session* s);

/* LlamaTransformer.Forward (src/model/llamatransformer.go:145-180) + the last-row
 * ml.Argmax of the generate loop (src/inference/inference.go:207-216).
 *   tokens[S] int32, start_pos as in the reference (S>1 requires start_pos==0, F11).
 *   logits : NULL, or host [S, vocab] f32 if all_rows, host [1, vocab] (last row) otherwise
 *   argmax_last : NULL, or receives the next token of the last row (greedy unless the sequence samples,
 *                 lnb_session_set_sampling).
 * One call = one H2D of tokens, the whole forward on the device, one D2H of what was asked. */
int lnb_forward(lnb_session* s, const int32_t* tokens, int S, int start_pos,
                float* logits, int all_rows, int32_t* argmax_last);

/* Batched decode (BASELINE.json configs[4], "concurrent prompts"): a session with n_seq (<= 8) independent
 * sequences = n_seq reference InferenceContexts sharing one set of weights (the reference has no batch
 * dimension, SURVEY F10).  lnb_session_set_active_sequence selects which sequence lnb_forward /
 * lnb_decode_run / lnb_session_read address (e.g. to prefill each prompt); lnb_forward_batch then advances
 * all sequences by one token in ONE pass over the weights: row i = sequence i, token tokens[i] at position
 * positions[i].  Every row gets exactly the arithmetic of its own S=1 Forward.  Any seq_len works: beyond
 * the shared-memory decode kernel's fit (351 positions at head_dim 128) the batched attention streams the
 * caches from HBM.  n_seq * seq_len positions of caches must fit the GPU, or creation is LNB_ENOMEM. */
int lnb_session_create_batch(lnb_model* m, int seq_len, int n_seq, int max_rows, int acc_mode, lnb_session** out);
int lnb_session_set_active_sequence(lnb_session* s, int seq);
int lnb_forward_batch(lnb_session* s, const int32_t* tokens, const int32_t* positions, int n,
                      float* logits /* NULL or [n, vocab] */,
                      int32_t* argmax_out /* [n]: next token (greedy unless the sequence samples) */);

/* LlamaTransformer.Forward whose result stays in HBM: the host mirror returns an ml.Tensor that carries a handle
 * (session, generation) instead of S x vocab floats, Tensor.Slice keeps the handle, and ml.Argmax on it runs on the
 * device -- the reference's call sequence Forward -> Slice(last row) -> Argmax (src/inference/inference.go:202-216)
 * moves 4 bytes per token over PCIe.  Touching the tensor's data calls lnb_session_logits_read.
 * rows_kept: 1 (last row) or S.  A handle is valid until the session's next forward (LNB_ESTATE afterwards).
 * Tensor-parallel: logits_read / logits_argmax are collectives (every rank makes the same call). */
int lnb_forward_device(lnb_session* s, const int32_t* tokens, int S, int start_pos, int rows_kept,
                       int32_t* argmax_last /* may be NULL; next token (greedy unless the sequence samples) */,
                       int64_t* generation_out);
/* lnb_session_logits_argmax is the greedy ml.Argmax of every row, sampled forward or not */
int lnb_session_logits_read(lnb_session* s, int64_t generation, int row0, int rows, float* host /* [rows, vocab] */);
int lnb_session_logits_argmax(lnb_session* s, int64_t generation, int row0, int rows, int32_t* out /* [rows] */);

/* EXTENSION beyond the reference (SURVEY 8f-4, chunked prefill): accept Forward calls of S > 1 tokens at startPos > 0 and
 * mask them with the [S,T] causal mask (row s sees keys t <= startPos + s).  The reference's [S,S] mask
 * (src/model/llamatransformer.go:128-136, added to [32,S,T] scores at :469-473) only broadcasts for startPos 0, which is
 * why the library refuses such calls by default, like the Go code would fail.  Chunked and one-shot prefill give
 * bit-identical caches and logits in LNB_ACC_STRICT. */
int lnb_session_set_chunked_prefill(lnb_session* s, int on);

/* EXTENSION (continuous batching): one forward over n_segs segments; segment i = len[i] tokens of sequence seq[i] at
 * positions start_pos[i] .. start_pos[i]+len[i]-1, rows laid out segment after segment in `tokens`.  Each segment gets the
 * arithmetic of its own Forward on its own InferenceContext (llamatransformer.go:145-180) under the [S,T] mask (row s sees
 * keys t <= start_pos + s; at start_pos 0 this is the reference's mask, :128-136), so prompts, prompt chunks and decode rows
 * of different sequences share one pass over the weights.
 *   valid: any session (single or batch); 1 <= n_segs <= n_seq; seq[] distinct, in [0, n_seq); len[i] >= 1,
 *   sum(len) <= max_rows; 0 <= start_pos[i], start_pos[i] + len[i] <= seq_len; token ids in range.  Anything else, and
 *   tp_size > 1 (not built), is LNB_EINVAL with nothing enqueued.  No lnb_session_set_chunked_prefill needed.
 *   logits: NULL or host [n_segs, vocab] f32, the LAST row of each segment; argmax_out: NULL or [n_segs], the next token
 *   of that row (greedy unless the sequence samples; greedy is inference.go:207-216).
 * Every ragged row's attention runs on the streamed kernels (csrc/sdpa_stream.cuh); LNB_ACC_FAST calls of >= 32 rows run
 * the projections on the tensor cores (one pass over the weights), all others the GEMV chain (one pass per 8 rows).
 * LNB_ACC_STRICT: every segment is bit-identical to its own Forward.  The first call allocates the row map and, if needed,
 * stream-attention scratch (LNB_ENOMEM with the bytes on failure; the session stays usable).  Afterwards a
 * lnb_forward_device handle is stale, the active sequence and a captured decode graph are unchanged, and
 * lnb_session_read(LNB_BUF_RESIDUAL) returns the call's [sum(len), dim] rows. */
int lnb_forward_ragged(lnb_session* s, int n_segs, const int32_t* seq, const int32_t* start_pos, const int32_t* len,
                       const int32_t* tokens, float* logits, int32_t* argmax_out);

/* EXTENSION: speculative verification.  Segment i = sequence seq[i], rows at positions start_pos[i] .. start_pos[i] + n_draft[i]:
 * row 0 feeds the sequence's last emitted token, rows 1.. feed the drafts (tokens: segment after segment, 1 + n_draft[i] ids each).
 * next_out[r] = the next token of row r (greedy, or sampled with p_next = its position + 1); n_accepted[i] = the largest a with
 * next_out[row j] == draft j+1 for all j < a.  The emitted tokens of segment i are next_out[its rows 0 .. a].
 * logits: NULL or host [rows, vocab].
 *   valid: any session (single or batch); 1 <= n_segs <= n_seq; seq[] distinct, in [0, n_seq); n_draft[i] >= 0;
 *   start_pos[i] >= 0, start_pos[i] + n_draft[i] < seq_len; total rows <= min(8, max_rows); token ids in range.  Anything
 *   else, and tp_size > 1 (not built), is LNB_EINVAL with nothing enqueued.  next_out / n_accepted may be NULL.
 *   Every row gets the arithmetic of its sequence's own S=1 Forward at its position: LNB_ACC_STRICT rows are bit-identical
 *   to it (and to the reference); LNB_ACC_FAST rows too on the batch engine's default form and, beyond the engines' limit,
 *   within the shared-memory decode kernel's fit (351 positions at head_dim 128).  Beyond that fit, and with
 *   LNB_BATCH_TC=1, FAST rows have the bits lnb_forward_batch gives those rows.  So a speculative stream is the plain stream.
 *   Routing: one row (one segment, no draft) is the ordinary S=1 step; >= 2 rows run ONE batch-engine launch when the session
 *   can run the engines (LNB_BATCH_ENGINE=0 opts out), else the kernel chain.
 *   Stale cache rows: the K/V rows of rejected drafts (positions start_pos + a + 1 and above) hold the drafts' keys and
 *   values.  Nothing reads them before the next call at start_pos + a + 1 overwrites them.
 *   Afterwards a lnb_forward_device handle is stale; the active sequence and a captured decode graph are unchanged (except
 *   that the first sampled call of more rows than the session has sequences grows the sampler's scratch, LNB_ENOMEM with the
 *   bytes on failure, and re-captures a sampled decode graph). */
int lnb_forward_speculative(lnb_session* s, int n_segs, const int32_t* seq, const int32_t* start_pos, const int32_t* n_draft,
                            const int32_t* tokens, float* logits, int32_t* next_out, int32_t* n_accepted);

/* Device-resident greedy decode: runs n_steps consecutive S=1 forwards starting with
 * `first_token` at position start_pos, feeding each argmax back on the device (no host
 * sync inside), optionally as CUDA-graph replays.  tokens_out[n_steps]; ms_out = device
 * time of the n_steps steps measured with CUDA events on the session stream.
 * This is the timed region of bench.py's `value`.  tokens_out: next token of each step (greedy unless the active sequence
 * samples; a sampled sequence decodes on the kernel chain with the sampler after each step, and lnb_last_error() says so
 * on a session whose S=1 steps otherwise run the persistent engine). */
int lnb_decode_run(lnb_session* s, int32_t first_token, int start_pos, int n_steps, int use_graph,
                   int32_t* tokens_out, float* ms_out);

/* EXTENSION (the reference's generate loop only has the greedy ml.Argmax, inference.go:207-216): seeded temperature,
 * top-k and top-p sampling, computed on the device (csrc/sample.cuh) with integer-exact arithmetic (DESIGN.md §9b).
 * For one row of logits l: the rank order is (l descending, index ascending); the candidates are the top_k first ranks
 * (0 or >= vocab: all); each gets the integer weight floor(2^40 exp(z)), z = f32(f32(l - max) / temperature), 0 for
 * z < -28; top_p keeps the shortest rank prefix of the candidates with at least ceil(top_p * their mass); the token is
 * drawn with 64 bits of splitmix64(seed, p_next), p_next = the position the token will occupy.  The draw depends only on
 * (row, parameters, p_next): a sequence's sampled stream does not depend on how it was batched, chunked or scheduled. */
typedef struct {
  float temperature;   /* 0: greedy; else finite, > 0 */
  int32_t top_k;       /* >= 0; 0: the whole vocabulary */
  float top_p;         /* (0, 1]; 1: no top-p cut */
  uint64_t seed;
} lnb_sampling;
/* Sequence `seq` of the session samples with *p from its next forward on; NULL or temperature 0: greedy (the default).
 * Every token output of the session's forwards for that sequence then carries the sampled token (lnb_forward /
 * lnb_forward_device argmax_last, lnb_forward_batch argmax_out, lnb_forward_ragged argmax_out, lnb_decode_run
 * tokens_out).  LNB_EINVAL with nothing changed: seq outside [0, n_seq), temperature not finite or < 0, top_k < 0,
 * top_p outside (0, 1], tp_size > 1 (not built).  The first sampler set allocates n_seq parameter slots and the weights
 * of n_seq rows (LNB_ENOMEM with the bytes; the session stays as it was).  Setting parameters does not synchronise the
 * stream or invalidate a captured decode graph; switching the active sequence between greedy and sampled re-captures it. */
int lnb_session_set_sampling(lnb_session* s, int seq, const lnb_sampling* p);

/* EXTENSION: repetition, frequency and presence penalties and a per-token logit bias, computed on the device
 * (csrc/penalty.cuh) over each sequence's token history, before the sampler (DESIGN.md §9e).  For the row that emits the
 * token at position p_next: c_t = how often token t was fed at positions [max(first_pos, p_next - window (0: no limit)),
 * p_next) of the sequence; where c_t >= 1, a = rp != 1 ? (l > 0 ? f32(l / rp) : f32(l * rp)) : l and
 * b = f32(a - f32(f32(f32(c_t) * fp) + pp)); then l' = f32(b + bias_t) for a biased token (-inf bias: l' = -inf, the token
 * is never emitted).  Every step is one rounded IEEE operation; a NaN a step produces is 0x7FFFFFFF (the device's NaN).
 * The sampler of lnb_session_set_sampling (greedy: rank 0) then runs unchanged on l', so a stream depends only on the
 * model, the prompt and the parameters, however it was batched, chunked or drafted.  Logprobs and the logits read-backs
 * keep reporting the raw distribution. */
#define LNB_LOGIT_BIAS_MAX 64
typedef struct {
  float repetition_penalty;   /* finite, > 0; 1: off */
  float frequency_penalty;    /* finite (may be negative); 0: off */
  float presence_penalty;     /* finite (may be negative); 0: off */
  int32_t window;             /* >= 0: count the last `window` positions; 0: every position */
  int32_t first_pos;          /* >= 0: positions below it are never counted (e.g. the prompt) */
  int32_t n_bias;             /* 0 .. LNB_LOGIT_BIAS_MAX */
  int32_t bias_token[LNB_LOGIT_BIAS_MAX];   /* distinct, in [0, vocab) */
  float bias[LNB_LOGIT_BIAS_MAX];           /* finite, or -inf (the token is never emitted) */
} lnb_penalties;
/* Sequence `seq` is penalized with *p from its next forward on; NULL or neutral parameters (rp 1, fp and pp 0, no bias)
 * turn penalties off (the default: the session launches exactly what it does without them).  Turning them on clears the
 * sequence's token history (stream-ordered); from then on every forward records the token of each of its rows at its
 * position, and every token the sequence emits is drawn from l'.  The first enable allocates the history of every sequence
 * and position (4 bytes each), the job's scratch and the sampler's slots (LNB_ENOMEM with the bytes; the session stays as
 * it was).  LNB_EINVAL with nothing changed: seq outside [0, n_seq), a parameter outside the ranges above, a bias token
 * repeated or outside [0, vocab), a +inf or NaN bias, tp_size > 1 (not built).  Turning penalties on or off for the active
 * sequence re-captures a decode graph; changing their values does not. */
int lnb_session_set_penalties(lnb_session* s, int seq, const lnb_penalties* p);

/* EXTENSION: token log-probabilities, computed on the device (csrc/logprob.cuh) and finished on the host (DESIGN.md §9d).
 * For one row of logits l and a token t: the rank order is the sampler's (l descending, index ascending), m the rank-0
 * logit, sum = the sum over the vocabulary of floor(2^40 exp(f32(l_i - m))) (0 below -28: the sampler's weights at
 * temperature 1, integers, so any reduction order gives the same bits), rank(t) = 1 + the tokens ranked before t, and
 * logprob(t) = (f64(l_t) - f64(m)) - log(f64(sum) 2^-40), within 1.2e-6 of the exact log-softmax at 128256 tokens.  The
 * logprob is always the raw model distribution (temperature 1, no top-k or top-p cut), also for sampled tokens.  A row
 * whose rank-0 logit is +inf or NaN gives NaN logprobs (rank 1 for its rank-0 token); a -inf logit gives -inf. */
#define LNB_LOGPROBS_TOP_MAX 20
typedef struct {
  int32_t token;     /* the scored token; -1: the position was never written */
  int32_t rank;      /* 1 = the greedy token */
  double logprob;
  int32_t n_top;     /* entries of top_token / top_logprob in use */
  int32_t top_token[LNB_LOGPROBS_TOP_MAX];   /* the n_top first tokens in rank order */
  double top_logprob[LNB_LOGPROBS_TOP_MAX];
} lnb_logprob;
/* top_n in [0, 20] turns logprobs on for sequence `seq` from its next forward on, -1 turns them off (the default).  Every
 * token a forward emits for that sequence (lnb_forward / lnb_forward_device argmax_last, lnb_forward_batch /
 * lnb_forward_ragged argmax_out, lnb_forward_speculative next_out, lnb_decode_run tokens_out; greedy or sampled) then writes
 * the record of the position it will occupy: record p of a sequence describes the token at position p given the tokens
 * before it, whatever the batching, chunking or scheduling.  Records of speculative rows beyond the accepted drafts, and of
 * ragged segments that end a non-final prompt chunk, describe tokens the caller discards: only positions whose token was
 * emitted or scored are meaningful (the stale-row rule of lnb_forward_speculative).  The first call that turns logprobs on
 * allocates records for every sequence and position, about 192 bytes each (LNB_ENOMEM with the bytes; the session stays as
 * it was).  LNB_EINVAL with nothing changed: seq outside [0, n_seq), top_n outside [-1, 20], tp_size > 1 (not built).
 * Turning logprobs on or off for the active sequence re-captures a decode graph; changing top_n does not. */
int lnb_session_set_logprobs(lnb_session* s, int seq, int top_n);
/* records [pos0, pos0 + n) of sequence `seq`, finished on the host, to out[n].  LNB_EINVAL: seq out of range, n < 1, or a
 * range outside [1, seq_len]. */
int lnb_session_logprobs_read(lnb_session* s, int seq, int pos0, int n, lnb_logprob* out);
/* Scoring: ONE forward of the active sequence over tokens[0 .. n-1) at positions start_pos .., with the LM head over all
 * those rows, then the records of positions start_pos + 1 .. start_pos + n - 1, whose tokens are tokens[1 .. n).  Chunked
 * scoring overlaps by one token: the next call starts at start_pos + n - 1 with tokens[n - 1].  2 <= n <= max_rows + 1,
 * start_pos + n <= seq_len + 1; start_pos > 0 needs lnb_session_set_chunked_prefill as lnb_forward does.  LNB_ESTATE when the
 * active sequence has logprobs off.  Afterwards a lnb_forward_device handle is stale. */
int lnb_score(lnb_session* s, const int32_t* tokens, int n, int start_pos);

/* EXTENSION: fork and permute sequences on the device (csrc/seqcopy.cuh, DESIGN.md §9f), e.g. for beam search.  For every
 * i < n, positions [pos0, pos1) of sequence dst[i] get what sequence src[i] held there BEFORE the call: K and V of every
 * layer, the penalty history (if allocated) and the logprob records (if allocated; record p is the token at position p).
 * The sources are read as a snapshot, so swaps, cycles and one source copied to many destinations are legal in one call;
 * a pair with src == dst is a no-op.  ONE stream-ordered launch (counted by lnb_session_launch_count), no host
 * synchronisation.  The active sequence, a lnb_forward_device logits handle and a captured decode graph stay valid.
 * Sampler and penalty parameters belong to the slot and are not copied: to fork a penalized sequence, enable penalties on
 * the destination first (enabling clears its history).  LNB_EINVAL with nothing enqueued: n outside [1, n_seq], dst[]
 * repeated or outside [0, n_seq), src[] outside [0, n_seq), not 0 <= pos0 < pos1 <= seq_len, more than 128 layers,
 * tp_size > 1 (not built). */
int lnb_session_copy_sequences(lnb_session* s, int n, const int32_t* src, const int32_t* dst, int pos0, int pos1);

/* Fused collective for tensor-parallel decode: instead of ncclAllReduce after Wo / w2, every rank's GEMV
 * epilogue stores its fp32 partials straight into all peers' memory over NVLink and a small kernel
 * reduces the N slots in rank order (bit-identical on every rank).  Setup: every rank exports the 64-byte
 * CUDA IPC handle of its session region, the host gathers the tp_size handles, every rank imports them
 * (index = rank).  Sessions must be created and driven identically on all ranks.  Without this call the
 * session uses NCCL (exactly one all-reduce after Wo and one after w2, as north_star prescribes). */
int lnb_session_p2p_export(lnb_session* s, void* handle64);
int lnb_session_p2p_import(lnb_session* s, const void* handles /* tp_size x 64 bytes */, int n);
/* Every in-kernel wait for a peer is bounded (LNB_P2P_TIMEOUT_MS, default 1500): a late or dead rank turns the
 * running call into LNB_ETIMEOUT on its peers instead of hanging their GPUs.  After that error the session's peer
 * path is poisoned; lnb_session_p2p_disable switches the session back to ncclAllReduce (all ranks must do the same). */
int lnb_session_p2p_disable(lnb_session* s);

/* debugging / parity probes */
enum { LNB_BUF_RESIDUAL = 0, LNB_BUF_CACHE_K = 1, LNB_BUF_CACHE_V = 2, LNB_BUF_LOGITS = 3 };
/* copies a device buffer of the session to host: RESIDUAL [S,dim] bf16 (after the last
 * forward; with lnb_session_set_layer_limit, after that many layers), CACHE_K/V of `layer`
 * [seq_len, n_kv_local, head_dim] bf16, LOGITS [rows, vocab_local] f32. */
int lnb_session_read(lnb_session* s, int which, int layer, void* host, int64_t nbytes);
int lnb_session_set_layer_limit(lnb_session* s, int n_layers_to_run); /* <=0: all */
/* Which decode path does the session use?  1 = the persistent decode engine (csrc/engine.cuh: one kernel launch runs n
 * complete S=1 forwards), 0 = the kernel chain (one launch per projection / attention / norm scale; lnb_last_error()
 * tells why).  LNB_ENGINE=1 / 0 forces the choice; the default is the engine except for single-GPU LNB_ACC_FAST. */
int lnb_session_decode_engine(lnb_session* s);
/* profiling aid of the persistent decode engine (LNB_ENGINE_PROF=1 when the session first decodes): cycles of consumer
 * thread 0 per section, {mean, max} over the CTAs, reset on read.  out[24]. */
int lnb_session_engine_profile(lnb_session* s, double* out16);
/* number of kernels launched by this session since creation (bench.py gpu_launches) */
int64_t lnb_session_launch_count(lnb_session* s);
int lnb_session_sync(lnb_session* s);
/* Measurement hook for bench.py's roofline: times ONE projection kernel of the decode step in
 * isolation (all layers' weights back to back so every launch streams from HBM; `reps` sweeps;
 * CUDA events on the session stream).  kind: 0 wq|wk|wv, 1 wo, 2 w1|w3, 3 w2, 4 LM head. */
int lnb_session_bench_kernel(lnb_session* s, int kind, int reps, float* ms_per_launch, int64_t* bytes_per_launch,
                             int* launches);

/* ------------------------------------------------------------------------------------
 * Op-level API -- what the src/ml shims bind.  Host pointers in and out; each call
 * stages through HBM and runs the same kernels the model path uses.
 * ---------------------------------------------------------------------------------- */

/* ml.LinearTransformation, BF16 (src/ml/operations_impl.go:427-447,
 * operations_lineartransform.go:37-70,145-207): x[S,K], w[N,K] -> out[S,N] */
int lnb_op_linear_bf16(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int K, int N, int acc_mode);
/* ml.MatMul, BF16 (operations_impl.go:449-476, operations_matmul.go:24-60,136-182):
 * a[B,M,K] x b[B,K,N] -> out[B,M,N] */
int lnb_op_matmul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int B, int M, int K, int N);
/* RMSNorm.Forward (src/model/llamatransformer.go:633-660) */
int lnb_op_rmsnorm_bf16(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int D, float eps, int acc_mode);
/* the scale of RMSNorm.Forward alone (llamatransformer.go:641-656: Pow, Mean, AddScalar, RSqrt):
 * r[s] = f32(1 / sqrt(f64( (sequential fp32 sum_k x[s,k]^2) / D + eps ))), bit-exact.
 * algo: 0 = what the model path uses (env LNB_RMS_ALGO=chain|scan|seg overrides the built-in choice),
 * 1 = one-thread FADD chain, 2 = iterative binade scan, 3 = one-pass predict / fold / walk
 * (csrc/seqsum.cuh; 2 and 3 return LNB_EINVAL when D does not fit their shape), 4 = the variant that runs inside the
 * persistent decode engine (256 threads, runs folded per warp; csrc/engine.cuh).  Identical bits. */
int lnb_op_rms_scale_f32(const uint16_t* x, float* r, int S, int D, float eps, int algo);
/* applyRotaryEmbeddings for one tensor (llamatransformer.go:753-790): x[S,H,hd] */
int lnb_op_rope_bf16(const uint16_t* x, const float* cis, uint16_t* out, int S, int H, int hd, int start_pos);
/* the attention core of LlamaAttention.Forward (llamatransformer.go:402-514):
 * q[S,n_heads,hd] rotated, cache_k/v[T,n_kv,hd] -> out[S,n_heads*hd].
 * causal_mask: 0 = none; 1 = the reference's [S,S] mask (T must equal S, LNB_EINVAL otherwise); 2 = EXTENSION, the
 * [S,T] mask of a chunked prefill: query row s sits at position T - S + s and sees the keys t <= T - S + s (the
 * kernels a session's chunked prefill runs for this mode and S) */
int lnb_op_attention_bf16(const uint16_t* q, const uint16_t* cache_k, const uint16_t* cache_v, uint16_t* out,
                          int S, int T, int n_heads, int n_kv, int hd, int causal_mask, int acc_mode);
/* ml.Silu (activations.go:27-50), ml.Add / ml.MultiplyElementwise same-shape bf16
 * (operations_impl.go:307-335,367-395) */
int lnb_op_silu_bf16(const uint16_t* x, uint16_t* out, int64_t n);
int lnb_op_add_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n);
int lnb_op_mul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n);
/* ml.Softmax on f32 rows (operations_impl.go:478-511), ml.Argmax (:513-548) */
int lnb_op_softmax_f32(const float* x, float* out, int rows, int cols);
int lnb_op_argmax_f32(const float* x, int rows, int cols, int32_t* out);
/* EXTENSION: the sampler of lnb_session_set_sampling alone on host rows (1..8 rows): logits[rows, vocab], parameters
 * p[rows], pos_next[rows] (the p_next of each draw) -> out[rows]; temperature 0 gives the greedy ml.Argmax (:513-548) */
int lnb_op_sample_f32(const float* logits, int rows, int vocab, const lnb_sampling* p, const int32_t* pos_next, int32_t* out);
/* EXTENSION: the logprob kernels of lnb_session_set_logprobs alone on host rows: logits[rows, vocab], targets[rows],
 * top_n in [0, 20] -> out[rows] */
int lnb_op_logprobs_f32(const float* logits, int rows, int vocab, const int32_t* targets, int top_n, lnb_logprob* out);
/* EXTENSION: the penalty kernels of lnb_session_set_penalties alone on host rows (1..8 rows): logits[rows, vocab],
 * parameters p[rows] (any valid parameters; a neutral row is copied), row r's token history hist[r][hist_len] (-1: not
 * counted), the position pos_next[r] in [0, hist_len] its token would occupy -> l' to out[rows, vocab] */
int lnb_op_penalize_f32(const float* logits, int rows, int vocab, const lnb_penalties* p, const int32_t* hist, int hist_len,
                        const int32_t* pos_next, float* out);
/* ml.Fwd_Get_Rows (operations_impl.go:142-173) */
int lnb_op_get_rows_bf16(const uint16_t* emb, const int32_t* tokens, uint16_t* out, int S, int vocab, int dim);

#ifdef __cplusplus
}
#endif
#endif /* LNB_H */
