// api.cu -- the C-ABI of liblnb.so (include/lnb.h): model / session lifecycle, the fused
// forward pass, the device-resident decode loop and the op-level entry points.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cerrno>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/lnb.h"
#include "gemm_tc.cuh"
#include "sdpa_tc.cuh"
#include "sdpa_stream.cuh"
#include "gemv.cuh"
#include "kernels.cuh"
#include "seqsum.cuh"
#include "engine.cuh"
#include "engine_batch.cuh"
#include "sample.cuh"
#include "logprob.cuh"
#include "penalty.cuh"
#include "seqcopy.cuh"
#include "pth.hpp"
#include "tokenizer.hpp"

namespace lnb {
void build_rope_table(int dim, int end, double theta, bool use_scaled, std::vector<float>& out);
void build_silu_table(std::vector<uint16_t>& out);
}  // namespace lnb

using namespace lnb;

// ------------------------------------------------------------------------------------------
// errors
static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return fail(LNB_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

extern "C" const char* lnb_last_error(void) { return g_err.c_str(); }
extern "C" int lnb_version(void) { return LNB_VERSION; }
extern "C" int lnb_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) return fail(LNB_ECUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
  return n;
}

// ------------------------------------------------------------------------------------------
// NCCL through dlopen (single-GPU use never needs the library)
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { ncclSum_ = 0, ncclMax_ = 2 };
enum { ncclUint64_ = 5, ncclFloat32_ = 7 };
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static std::mutex g_nccl_mu;
static int nccl_load() {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.h) return 0;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.h) break;
  }
  if (!g_nccl.h) return fail(LNB_ENCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
#define SYM(field, name)                                                  \
  *(void**)(&g_nccl.field) = dlsym(g_nccl.h, name);                       \
  if (!g_nccl.field) return fail(LNB_ENCCL, "libnccl lacks %s", name);
  SYM(GetUniqueId, "ncclGetUniqueId");
  SYM(CommInitRank, "ncclCommInitRank");
  SYM(CommDestroy, "ncclCommDestroy");
  SYM(AllReduce, "ncclAllReduce");
  SYM(AllGather, "ncclAllGather");
  SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
  return 0;
}
#define NC(call)                                                                                \
  do {                                                                                          \
    int r_ = (call);                                                                            \
    if (r_ != 0) return fail(LNB_ENCCL, "%s failed: %s", #call, g_nccl.GetErrorString(r_));     \
  } while (0)

extern "C" int lnb_nccl_unique_id(void* out128) {
  if (!out128) return fail(LNB_EINVAL, "out128 is NULL");
  int rc = nccl_load();
  if (rc) return rc;
  ncclUniqueId id;
  NC(g_nccl.GetUniqueId(&id));
  memcpy(out128, &id, 128);
  return 0;
}

// ------------------------------------------------------------------------------------------
// model
struct LayerW {
  uint16_t *attn_norm = nullptr, *wqkv = nullptr, *wo = nullptr, *ffn_norm = nullptr, *w13 = nullptr, *w2 = nullptr;
  unsigned have = 0;  // bit per checkpoint tensor (9)
};
enum { T_ATTN_NORM = 0, T_WQ, T_WK, T_WV, T_WO, T_FFN_NORM, T_W1, T_W2, T_W3, T_EMBD, T_NORM, T_OUTPUT };

struct lnb_model {
  lnb_model_args a;
  int device = 0, tp_rank = 0, tp_size = 1;
  int q_dim = 0, kv_dim = 0, q_l = 0, kv_l = 0, ffn_l = 0, vocab_l = 0;
  uint16_t *tok_embd = nullptr, *norm = nullptr, *output = nullptr;
  bool have_embd = false, have_norm = false, have_output = false, finalized = false;
  std::vector<LayerW> layers;
  float* cis = nullptr;
  int cis_rows = 0;
  uint16_t* silu_tab = nullptr;
  bool cis_set = false, silu_set = false;
  ncclComm_t comm = nullptr;
  void* staging = nullptr;
  size_t staging_bytes = 0;
  int sm_count = 132;
  // the STRICT decode engine's packed copies of w1|w3 (per layer) and the LM head (wpack.cuh), built by the first STRICT
  // engine session (ensure_wpack).  Sessions need a finalized model and a finalized model takes no more weights, so a
  // packed copy can never fall behind the bf16 matrix it was built from.
  struct WPack {
    uint8_t* data = nullptr;
    uint8_t* units = nullptr;
    int kt = 0;
    int64_t read_bytes = 0;        // bytes the engine reads per pass (packed units, raw units, unit table)
    int64_t packed_units = 0, n_units = 0;
  };
  std::vector<WPack> wp_w13;
  WPack wp_out;
  void* wpack_mem = nullptr;
  int wpack_state = 0;             // 0 = not built, 1 = built, -1 = the engine streams bf16 (wpack_why says why)
  std::string wpack_why;
  std::mutex wpack_mu;
};

static int parse_name(const lnb_model* m, const char* name, int* kind, int* layer) {
  *layer = -1;
  if (!strcmp(name, "tok_embeddings.weight")) { *kind = T_EMBD; return 0; }
  if (!strcmp(name, "norm.weight")) { *kind = T_NORM; return 0; }
  if (!strcmp(name, "output.weight")) { *kind = T_OUTPUT; return 0; }
  int l = -1;
  char rest[96];
  if (sscanf(name, "layers.%d.%95s", &l, rest) != 2 || l < 0 || l >= m->a.n_layers) return -1;
  *layer = l;
  static const char* names[9] = {"attention_norm.weight", "attention.wq.weight", "attention.wk.weight",
                                 "attention.wv.weight",   "attention.wo.weight", "ffn_norm.weight",
                                 "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight"};
  for (int i = 0; i < 9; i++)
    if (!strcmp(rest, names[i])) { *kind = i; return 0; }
  return -1;
}

// full checkpoint shape of a tensor kind (llamatransformer.go:84-105,191,202,273-282,580-586)
static void full_shape(const lnb_model* m, int kind, int64_t* rows, int64_t* cols) {
  const lnb_model_args& a = m->a;
  switch (kind) {
    case T_ATTN_NORM: case T_FFN_NORM: case T_NORM: *rows = a.dim; *cols = 1; break;
    case T_WQ: *rows = m->q_dim; *cols = a.dim; break;
    case T_WK: case T_WV: *rows = m->kv_dim; *cols = a.dim; break;
    case T_WO: *rows = a.dim; *cols = m->q_dim; break;
    case T_W1: case T_W3: *rows = a.ffn_dim; *cols = a.dim; break;
    case T_W2: *rows = a.dim; *cols = a.ffn_dim; break;
    case T_EMBD: case T_OUTPUT: *rows = a.vocab_size; *cols = a.dim; break;
  }
}

// where a checkpoint tensor lands in the HBM layout of this rank
struct Placement {
  uint16_t* dst;
  int64_t row0, col0;  // window of the full tensor owned by this rank
  int rows, cols;      // window size
  bool panel_major;
  int dpanel0, dpanel_stride;
};
static Placement placement(lnb_model* m, int kind, int layer) {
  Placement p{};
  const lnb_model_args& a = m->a;
  const int r = m->tp_rank;
  p.dpanel0 = 0;
  p.dpanel_stride = 1;
  p.panel_major = true;
  LayerW* L = layer >= 0 ? &m->layers[layer] : nullptr;
  switch (kind) {
    case T_ATTN_NORM: p.dst = L->attn_norm; p.rows = 1; p.cols = a.dim; p.panel_major = false; break;
    case T_FFN_NORM: p.dst = L->ffn_norm; p.rows = 1; p.cols = a.dim; p.panel_major = false; break;
    case T_NORM: p.dst = m->norm; p.rows = 1; p.cols = a.dim; p.panel_major = false; break;
    case T_EMBD: p.dst = m->tok_embd; p.rows = a.vocab_size; p.cols = a.dim; p.panel_major = false; break;
    case T_WQ: p.dst = L->wqkv; p.row0 = (int64_t)r * m->q_l; p.rows = m->q_l; p.cols = a.dim; break;
    case T_WK: p.dst = L->wqkv; p.row0 = (int64_t)r * m->kv_l; p.rows = m->kv_l; p.cols = a.dim; p.dpanel0 = m->q_l / 8; break;
    case T_WV: p.dst = L->wqkv; p.row0 = (int64_t)r * m->kv_l; p.rows = m->kv_l; p.cols = a.dim; p.dpanel0 = (m->q_l + m->kv_l) / 8; break;
    case T_WO: p.dst = L->wo; p.col0 = (int64_t)r * m->q_l; p.rows = a.dim; p.cols = m->q_l; break;
    case T_W1: p.dst = L->w13; p.row0 = (int64_t)r * m->ffn_l; p.rows = m->ffn_l; p.cols = a.dim; p.dpanel0 = 0; p.dpanel_stride = 2; break;
    case T_W3: p.dst = L->w13; p.row0 = (int64_t)r * m->ffn_l; p.rows = m->ffn_l; p.cols = a.dim; p.dpanel0 = 2; p.dpanel_stride = 2; break;
    case T_W2: p.dst = L->w2; p.col0 = (int64_t)r * m->ffn_l; p.rows = a.dim; p.cols = m->ffn_l; break;
    case T_OUTPUT: p.dst = m->output; p.row0 = (int64_t)r * m->vocab_l; p.rows = m->vocab_l; p.cols = a.dim; break;
  }
  return p;
}

static void mark_present(lnb_model* m, int kind, int layer) {
  if (kind == T_EMBD) m->have_embd = true;
  else if (kind == T_NORM) m->have_norm = true;
  else if (kind == T_OUTPUT) m->have_output = true;
  else m->layers[layer].have |= 1u << kind;
}

// Pure host arithmetic (no CUDA): which window of checkpoint tensor `name` rank tp_rank owns.
extern "C" int lnb_tp_shard_window(const lnb_model_args* args, const char* name, int tp_rank, int tp_size,
                                   int64_t* row0, int64_t* col0, int64_t* rows, int64_t* cols) {
  if (!args || !name || !row0 || !col0 || !rows || !cols) return fail(LNB_EINVAL, "NULL argument");
  if (tp_size < 1 || tp_rank < 0 || tp_rank >= tp_size) return fail(LNB_EINVAL, "bad tp rank %d / size %d", tp_rank, tp_size);
  const lnb_model_args& a = *args;
  if (a.n_kv_heads % tp_size || a.ffn_dim % tp_size || a.vocab_size % tp_size)
    return fail(LNB_EINVAL, "tp_size %d must divide n_kv_heads, ffn_dim and vocab_size", tp_size);
  lnb_model tmp;
  tmp.a = a;
  tmp.tp_rank = tp_rank;
  tmp.tp_size = tp_size;
  tmp.q_dim = a.n_heads * a.head_dim;
  tmp.kv_dim = a.n_kv_heads * a.head_dim;
  tmp.q_l = tmp.q_dim / tp_size;
  tmp.kv_l = tmp.kv_dim / tp_size;
  tmp.ffn_l = a.ffn_dim / tp_size;
  tmp.vocab_l = a.vocab_size / tp_size;
  tmp.layers.resize(a.n_layers);
  int kind, layer;
  if (parse_name(&tmp, name, &kind, &layer)) return fail(LNB_EINVAL, "unknown tensor name \"%s\"", name);
  Placement p = placement(&tmp, kind, layer);
  int64_t fr, fc;
  full_shape(&tmp, kind, &fr, &fc);
  *row0 = p.row0; *col0 = p.col0;
  if (fc == 1) { *rows = fr; *cols = 1; }  // 1-D tensors are replicated
  else { *rows = p.rows; *cols = p.cols; }
  return 0;
}

extern "C" int lnb_model_create(const lnb_model_args* args, int device, int tp_rank, int tp_size,
                                const void* nccl_unique_id, lnb_model** out) {
  if (!args || !out) return fail(LNB_EINVAL, "args/out is NULL");
  const lnb_model_args& a = *args;
  if (a.dim <= 0 || a.n_layers <= 0 || a.n_heads <= 0 || a.n_kv_heads <= 0 || a.head_dim <= 0 || a.ffn_dim <= 0 ||
      a.vocab_size <= 0 || a.max_seq_len <= 0)
    return fail(LNB_EINVAL, "non-positive model dimension");
  if (a.n_heads % a.n_kv_heads) return fail(LNB_EINVAL, "n_heads %d not a multiple of n_kv_heads %d", a.n_heads, a.n_kv_heads);
  // every attention kernel reads a head's K/V row as 16-byte vectors (8 bf16) from cache + t * kv_dim + h * head_dim
  if (a.head_dim % 8) return fail(LNB_EINVAL, "head_dim %d must be a multiple of 8 (the attention kernels read K/V rows 8 elements at a time)", a.head_dim);
  if (tp_size < 1 || tp_rank < 0 || tp_rank >= tp_size) return fail(LNB_EINVAL, "bad tp rank %d / size %d", tp_rank, tp_size);
  if (a.n_kv_heads % tp_size || a.ffn_dim % tp_size || a.vocab_size % tp_size)
    return fail(LNB_EINVAL, "tp_size %d must divide n_kv_heads, ffn_dim and vocab_size", tp_size);
  const int q_dim = a.n_heads * a.head_dim, kv_dim = a.n_kv_heads * a.head_dim;
  const int q_l = q_dim / tp_size, kv_l = kv_dim / tp_size, ffn_l = a.ffn_dim / tp_size, vocab_l = a.vocab_size / tp_size;
  if (a.dim % 32 || q_l % 32 || kv_l % 32 || ffn_l % 16 || vocab_l % 16)
    return fail(LNB_EINVAL, "dimension not tileable: dim %d q_l %d kv_l %d ffn_l %d vocab_l %d (need multiples of 32/32/32/16/16)",
                a.dim, q_l, kv_l, ffn_l, vocab_l);
  if (tp_size > 1 && !nccl_unique_id) return fail(LNB_EINVAL, "tp_size>1 needs an nccl unique id");
  CU(cudaSetDevice(device));
  lnb_model* m = new lnb_model();
  m->a = a;
  m->device = device;
  m->tp_rank = tp_rank;
  m->tp_size = tp_size;
  m->q_dim = q_dim; m->kv_dim = kv_dim; m->q_l = q_l; m->kv_l = kv_l; m->ffn_l = ffn_l; m->vocab_l = vocab_l;
  cudaDeviceGetAttribute(&m->sm_count, cudaDevAttrMultiProcessorCount, device);
  m->layers.resize(a.n_layers);
  auto alloc16 = [&](uint16_t** p, size_t elems) -> cudaError_t { return cudaMalloc((void**)p, elems * 2); };
  cudaError_t e = cudaSuccess;
  e = alloc16(&m->tok_embd, (size_t)a.vocab_size * a.dim);
  if (e == cudaSuccess) e = alloc16(&m->norm, a.dim);
  if (e == cudaSuccess) e = alloc16(&m->output, (size_t)vocab_l * a.dim);
  for (int l = 0; l < a.n_layers && e == cudaSuccess; l++) {
    LayerW& L = m->layers[l];
    e = alloc16(&L.attn_norm, a.dim);
    if (e == cudaSuccess) e = alloc16(&L.ffn_norm, a.dim);
    if (e == cudaSuccess) e = alloc16(&L.wqkv, (size_t)(q_l + 2 * kv_l) * a.dim);
    if (e == cudaSuccess) e = alloc16(&L.wo, (size_t)a.dim * q_l);
    if (e == cudaSuccess) e = alloc16(&L.w13, (size_t)2 * ffn_l * a.dim);
    if (e == cudaSuccess) e = alloc16(&L.w2, (size_t)a.dim * ffn_l);
  }
  if (e == cudaSuccess) e = cudaMalloc((void**)&m->silu_tab, 65536 * 2);
  if (e != cudaSuccess) {
    lnb_model_destroy(m);
    return fail(LNB_ENOMEM, "cudaMalloc of model weights failed: %s", cudaGetErrorString(e));
  }
  if (tp_size > 1) {
    int rc = nccl_load();
    if (rc) { lnb_model_destroy(m); return rc; }
    ncclUniqueId id;
    memcpy(&id, nccl_unique_id, 128);
    int r = g_nccl.CommInitRank(&m->comm, tp_size, id, tp_rank);
    if (r != 0) { lnb_model_destroy(m); return fail(LNB_ENCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString(r)); }
  }
  *out = m;
  return 0;
}

extern "C" int lnb_model_destroy(lnb_model* m) {
  if (!m) return 0;
  cudaSetDevice(m->device);
  cudaDeviceSynchronize();
  if (m->comm) g_nccl.CommDestroy(m->comm);
  cudaFree(m->tok_embd); cudaFree(m->norm); cudaFree(m->output);
  for (auto& L : m->layers) {
    cudaFree(L.attn_norm); cudaFree(L.ffn_norm); cudaFree(L.wqkv); cudaFree(L.wo); cudaFree(L.w13); cudaFree(L.w2);
  }
  cudaFree(m->cis); cudaFree(m->silu_tab); cudaFree(m->staging); cudaFree(m->wpack_mem);
  delete m;
  return 0;
}

static int ensure_staging(lnb_model* m, size_t bytes) {
  if (m->staging_bytes >= bytes) return 0;
  if (m->staging) cudaFree(m->staging);
  m->staging = nullptr;
  m->staging_bytes = 0;
  CU(cudaMalloc(&m->staging, bytes));
  m->staging_bytes = bytes;
  return 0;
}

extern "C" int lnb_model_upload_tensor(lnb_model* m, const char* name, const uint16_t* host, const int64_t* shape, int ndim) {
  if (!m || !name || !host || !shape) return fail(LNB_EINVAL, "NULL argument");
  if (m->finalized) return fail(LNB_ESTATE, "model is finalized");
  int kind, layer;
  if (parse_name(m, name, &kind, &layer)) return fail(LNB_EINVAL, "unknown tensor name \"%s\"", name);
  int64_t rows, cols;
  full_shape(m, kind, &rows, &cols);
  // same check as getTensor (src/model/loader.go:183-197)
  bool ok = (cols == 1) ? (ndim == 1 && shape[0] == rows) : (ndim == 2 && shape[0] == rows && shape[1] == cols);
  if (!ok) return fail(LNB_EINVAL, "tensor \"%s\": unexpected shape (expected [%lld%s%lld])", name, (long long)rows,
                       cols == 1 ? "] / [" : ", ", (long long)cols);
  CU(cudaSetDevice(m->device));
  Placement p = placement(m, kind, layer);
  const int64_t ld = (cols == 1) ? rows : cols;
  if (!p.panel_major) {
    CU(cudaMemcpy(p.dst, host, (size_t)p.rows * p.cols * 2, cudaMemcpyHostToDevice));
  } else {
    int rc = ensure_staging(m, (size_t)p.rows * p.cols * 2);
    if (rc) return rc;
    CU(cudaMemcpy2D(m->staging, (size_t)p.cols * 2, host + p.row0 * ld + p.col0, (size_t)ld * 2, (size_t)p.cols * 2,
                    p.rows, cudaMemcpyHostToDevice));
    retile_kernel<<<m->sm_count * 8, 256>>>((const uint16_t*)m->staging, p.cols, 0, 0, p.rows, p.cols, p.dst, p.dpanel0,
                                            p.dpanel_stride);
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
  }
  mark_present(m, kind, layer);
  return 0;
}

// ---- checkpoint files (SURVEY 8f-1): .pth reader / writer, params.json --------------------------
struct lnb_pth {
  lnb::PthFile f;
};
struct lnb_pth_writer {
  lnb::PthWriter w;
};

extern "C" int lnb_pth_open(const char* path, lnb_pth** out) {
  if (!path || !out) return fail(LNB_EINVAL, "NULL argument");
  lnb_pth* h = new lnb_pth();
  std::string err;
  if (!h->f.open(path, err)) {
    delete h;
    return fail(LNB_EINVAL, "%s", err.c_str());
  }
  *out = h;
  return 0;
}
extern "C" int lnb_pth_close(lnb_pth* f) {
  delete f;
  return 0;
}
extern "C" int lnb_pth_tensor_count(const lnb_pth* f) {
  if (!f) return fail(LNB_EINVAL, "NULL argument");
  return (int)f->f.tensors().size();
}
extern "C" int lnb_pth_tensor_info(const lnb_pth* f, int index, const char** name, int* dtype, int* ndim, int64_t* shape,
                                   int64_t* file_offset, int64_t* nbytes) {
  if (!f) return fail(LNB_EINVAL, "NULL argument");
  if (index < 0 || index >= (int)f->f.tensors().size()) return fail(LNB_EINVAL, "tensor index %d out of range", index);
  const lnb::PthTensor& t = f->f.tensors()[index];
  if (t.shape.size() > 8) return fail(LNB_EINVAL, "tensor \"%s\" has more than 8 dimensions", t.name.c_str());
  if (name) *name = t.name.c_str();
  if (dtype) *dtype = t.dtype;
  if (ndim) *ndim = (int)t.shape.size();
  if (shape) for (size_t i = 0; i < t.shape.size(); i++) shape[i] = t.shape[i];
  if (file_offset) *file_offset = t.file_offset;
  if (nbytes) *nbytes = t.nbytes;
  return t.contiguous ? 0 : 1;
}
extern "C" const void* lnb_pth_tensor_data(const lnb_pth* f, int index) {
  if (!f || index < 0 || index >= (int)f->f.tensors().size()) {
    fail(LNB_EINVAL, "tensor index %d out of range", index);
    return nullptr;
  }
  return f->f.data(f->f.tensors()[index]);
}

// torch.NewTorchModelReader + Load + the name / shape binding of NewLlamaTransformer, in one pass over the
// mapping: every tensor the architecture names is copied (TP: sliced) from the page cache into HBM.
extern "C" int lnb_model_load_pth(lnb_model* m, const char* path, int* n_uploaded) {
  if (!m || !path) return fail(LNB_EINVAL, "NULL argument");
  if (m->finalized) return fail(LNB_ESTATE, "model is finalized");
  lnb::PthFile f;
  std::string err;
  if (!f.open(path, err)) return fail(LNB_EINVAL, "%s", err.c_str());
  int n = 0;
  for (const lnb::PthTensor& t : f.tensors()) {
    int kind, layer;
    if (parse_name(m, t.name.c_str(), &kind, &layer)) continue;   // e.g. "rope.freqs": the reference never asks for it either
    if (t.dtype != lnb::PTH_BF16)
      return fail(LNB_EINVAL, "tensor \"%s\" is %s; the reference reads torch.BFloat16Storage only (src/torch/types.go:9-21)", t.name.c_str(),
                  lnb::pth_dtype_name(t.dtype));
    if (!t.contiguous) return fail(LNB_EINVAL, "tensor \"%s\" is not contiguous", t.name.c_str());
    if (t.shape.size() > 2) return fail(LNB_EINVAL, "tensor \"%s\": unexpected rank %zu", t.name.c_str(), t.shape.size());
    int rc = lnb_model_upload_tensor(m, t.name.c_str(), (const uint16_t*)f.data(t), t.shape.data(), (int)t.shape.size());
    if (rc) return rc;
    n++;
  }
  if (n_uploaded) *n_uploaded = n;
  return 0;
}

// loadModelArgsFromFile (src/model/modelargs.go:52-64) + the derived fields (llamatransformer.go:73-82,569-577)
extern "C" int lnb_model_args_from_params_json(const char* path, int max_seq_len, lnb_model_args* out) {
  if (!path || !out) return fail(LNB_EINVAL, "NULL argument");
  FILE* fp = fopen(path, "rb");
  if (!fp) return fail(LNB_EINVAL, "open %s: %s", path, strerror(errno));
  std::string text;
  char buf[4096];
  size_t k;
  while ((k = fread(buf, 1, sizeof(buf), fp)) > 0) text.append(buf, k);
  fclose(fp);
  lnb::ParamsJson pj;
  std::string err;
  if (!lnb::parse_params_json(text, pj, err)) return fail(LNB_EINVAL, "%s", err.c_str());
  if (pj.dim <= 0 || pj.n_heads <= 0 || pj.multiple_of <= 0) return fail(LNB_EINVAL, "params.json: non-positive dimension");
  lnb_model_args a{};
  a.dim = pj.dim;
  a.n_layers = pj.n_layers;
  a.n_heads = pj.n_heads;
  a.n_kv_heads = pj.n_kv_heads < 0 ? pj.n_heads : pj.n_kv_heads;
  a.head_dim = pj.dim / pj.n_heads;
  int hidden = 4 * pj.dim;
  hidden = (int)(2 * hidden / 3);
  if (pj.ffn_dim_multiplier > -1) hidden = (int)(pj.ffn_dim_multiplier * (double)hidden);
  a.ffn_dim = pj.multiple_of * ((hidden + pj.multiple_of - 1) / pj.multiple_of);
  a.vocab_size = pj.vocab_size;          // -1 when absent: the reference takes it from the tokenizer (loader.go:108-110)
  a.max_seq_len = max_seq_len > 0 ? max_seq_len : 2048;
  a.norm_eps = pj.norm_eps;
  a.rope_theta = pj.rope_theta > 0 ? pj.rope_theta : 500000.0;
  a.use_scaled_rope = pj.use_scaled_rope ? 1 : 0;
  *out = a;
  return 0;
}

extern "C" int lnb_pth_writer_create(const char* path, lnb_pth_writer** out) {
  if (!path || !out) return fail(LNB_EINVAL, "NULL argument");
  lnb_pth_writer* w = new lnb_pth_writer();
  std::string err;
  if (!w->w.open(path, err)) {
    delete w;
    return fail(LNB_EINVAL, "%s", err.c_str());
  }
  *out = w;
  return 0;
}
extern "C" int lnb_pth_writer_add(lnb_pth_writer* w, const char* name, int dtype, const void* data, const int64_t* shape, int ndim) {
  if (!w || !name || (!data && ndim > 0) || (!shape && ndim > 0)) return fail(LNB_EINVAL, "NULL argument");
  if (ndim < 0 || ndim > 8) return fail(LNB_EINVAL, "bad rank %d", ndim);
  std::string err;
  std::vector<int64_t> sh(shape, shape + ndim);
  if (!w->w.add(name, dtype, data, sh, err)) return fail(LNB_EINVAL, "%s", err.c_str());
  return 0;
}
extern "C" int lnb_pth_writer_finish(lnb_pth_writer* w) {
  if (!w) return fail(LNB_EINVAL, "NULL argument");
  std::string err;
  const bool ok = w->w.finish(err);
  delete w;
  return ok ? 0 : fail(LNB_EINVAL, "%s", err.c_str());
}

// ---- tokenizer (SURVEY 8f-3): tiktoken vocabulary + BPE, host-only ----------------------------------
struct lnb_vocab {
  lnb::Vocab v;
};
extern "C" int lnb_vocab_load(const char* tokenizer_model_path, lnb_vocab** out) {
  if (!tokenizer_model_path || !out) return fail(LNB_EINVAL, "NULL argument");
  lnb_vocab* h = new lnb_vocab();
  std::string err;
  if (!h->v.load(tokenizer_model_path, err)) {
    delete h;
    return fail(LNB_EINVAL, "%s", err.c_str());
  }
  *out = h;
  return 0;
}
extern "C" int lnb_vocab_write_synthetic(const char* path, int n_mergeable) {
  if (!path) return fail(LNB_EINVAL, "NULL argument");
  std::string err;
  if (!lnb::write_synthetic_vocab(path, n_mergeable, err)) return fail(LNB_EINVAL, "%s", err.c_str());
  return 0;
}
extern "C" int lnb_vocab_destroy(lnb_vocab* v) {
  delete v;
  return 0;
}
extern "C" int lnb_vocab_size(const lnb_vocab* v) {
  if (!v) return fail(LNB_EINVAL, "NULL argument");
  return v->v.size();
}
extern "C" int lnb_vocab_token_id(const lnb_vocab* v, const void* token, int token_len, int32_t* id) {
  if (!v || !token || token_len < 0 || !id) return fail(LNB_EINVAL, "bad argument");
  *id = v->v.id_of(std::string((const char*)token, (size_t)token_len));
  return 0;
}
extern "C" int lnb_vocab_token_bytes(const lnb_vocab* v, int32_t id, const void** bytes, int* len) {
  if (!v || !bytes || !len) return fail(LNB_EINVAL, "NULL argument");
  if (id < 0 || id >= v->v.size()) return fail(LNB_EINVAL, "token id %d out of range", id);
  *bytes = v->v.id_to_token[(size_t)id].data();
  *len = (int)v->v.id_to_token[(size_t)id].size();
  return 0;
}
extern "C" int lnb_vocab_special_ids(const lnb_vocab* v, int32_t* bos, int32_t* eos, int32_t* pad, int32_t* stop2) {
  if (!v) return fail(LNB_EINVAL, "NULL argument");
  if (bos) *bos = v->v.bos_id;
  if (eos) *eos = v->v.eos_id;
  if (pad) *pad = v->v.pad_id;
  if (stop2) { stop2[0] = v->v.stop_ids[0]; stop2[1] = v->v.stop_ids[1]; }
  return 0;
}
static int copy_ids(const std::vector<int32_t>& ids, int32_t* out, int cap, int* n_out) {
  if (n_out) *n_out = (int)ids.size();
  if ((int)ids.size() > cap) return fail(LNB_EINVAL, "token buffer too small: need %zu, have %d", ids.size(), cap);
  if (!ids.empty()) memcpy(out, ids.data(), ids.size() * 4);
  return 0;
}
extern "C" int lnb_tokenize_string(const lnb_vocab* v, const char* text, int64_t text_len, int32_t* out, int cap, int* n_out) {
  if (!v || (!text && text_len > 0) || text_len < 0 || (!out && cap > 0)) return fail(LNB_EINVAL, "bad argument");
  std::vector<int32_t> ids;
  v->v.tokenize_string(std::string(text ? text : "", (size_t)text_len), ids);
  return copy_ids(ids, out, cap, n_out);
}
extern "C" int lnb_split_pieces(const char* text, int64_t text_len, int64_t* ends, int cap, int* n_out) {
  if ((!text && text_len > 0) || text_len < 0 || (!ends && cap > 0)) return fail(LNB_EINVAL, "bad argument");
  const std::string t(text ? text : "", (size_t)text_len);
  int n = 0;
  for (size_t p = 0; p < t.size();) {
    p = lnb::Vocab::next_piece(t, p);
    if (n < cap) ends[n] = (int64_t)p;
    n++;
  }
  if (n_out) *n_out = n;
  return n > cap ? fail(LNB_EINVAL, "piece buffer too small: need %d, have %d", n, cap) : 0;
}
extern "C" int lnb_tokenize_prompt(const lnb_vocab* v, const char* const* headers, const char* const* contents, int n_parts,
                                   int32_t* out, int cap, int* n_out) {
  if (!v || n_parts < 0 || (n_parts > 0 && (!headers || !contents)) || (!out && cap > 0)) return fail(LNB_EINVAL, "bad argument");
  std::vector<lnb::PromptPart> parts;
  for (int i = 0; i < n_parts; i++) {
    if (!headers[i] || !contents[i]) return fail(LNB_EINVAL, "NULL prompt part");
    parts.push_back(lnb::PromptPart{headers[i], contents[i]});
  }
  std::vector<int32_t> ids;
  std::string err;
  if (!v->v.tokenize_prompt(parts, ids, err)) return fail(LNB_EINVAL, "%s", err.c_str());
  return copy_ids(ids, out, cap, n_out);
}
extern "C" int lnb_detokenize(const lnb_vocab* v, const int32_t* ids, int n, char* out, int64_t cap, int64_t* n_out) {
  if (!v || (!ids && n > 0) || n < 0 || (!out && cap > 0)) return fail(LNB_EINVAL, "bad argument");
  std::string s;
  if (!v->v.detokenize(ids, n, s)) return fail(LNB_EINVAL, "token id out of range");
  if (n_out) *n_out = (int64_t)s.size();
  if ((int64_t)s.size() > cap) return fail(LNB_EINVAL, "text buffer too small: need %zu", s.size());
  if (!s.empty()) memcpy(out, s.data(), s.size());
  return 0;
}

// ---- synthetic checkpoint ------------------------------------------------------------------
static uint64_t fnv1a64(const char* s) {
  uint64_t h = 0xcbf29ce484222325ULL;
  for (; *s; s++) { h ^= (uint8_t)*s; h *= 0x100000001b3ULL; }
  return h;
}
static void synth_spec_kind(const lnb_model_args& a, int kind, float* scale, float* offset) {
  const float s3 = 1.7320508075688772f;
  *offset = 0.f;
  switch (kind) {
    case T_EMBD: *scale = 1.0f; break;
    case T_ATTN_NORM: case T_FFN_NORM: case T_NORM: *scale = 0.1f; *offset = 1.0f; break;
    case T_W2: *scale = s3 / sqrtf((float)a.ffn_dim); break;
    case T_OUTPUT: *scale = 0.25f * s3 / sqrtf((float)a.dim); break;
    case T_WO: *scale = s3 / sqrtf((float)(a.n_heads * a.head_dim)); break;
    default: *scale = s3 / sqrtf((float)a.dim); break;
  }
}
extern "C" int lnb_synth_spec(const lnb_model_args* args, const char* name, float* scale, float* offset) {
  if (!args || !name || !scale || !offset) return fail(LNB_EINVAL, "NULL argument");
  lnb_model tmp;
  tmp.a = *args;
  int kind, layer;
  if (parse_name(&tmp, name, &kind, &layer)) return fail(LNB_EINVAL, "unknown tensor name \"%s\"", name);
  synth_spec_kind(*args, kind, scale, offset);
  return 0;
}
static void synth_fill_range(uint64_t s, float scale, float offset, int64_t i0, int64_t i1, uint16_t* out) {
  for (int64_t i = i0; i < i1; i++) {
    uint64_t z = s + ((uint64_t)i + 1) * 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z = z ^ (z >> 31);
    volatile float u = (float)(z >> 40) * (1.0f / 16777216.0f);
    volatile float w = 2.0f * u - 1.0f;
    volatile float v = w * scale;
    volatile float v2 = v + offset;
    float vv = v2;
    uint32_t b;
    memcpy(&b, &vv, 4);
    out[i] = (uint16_t)(b >> 16);
  }
}
extern "C" int lnb_synth_fill_host(uint64_t seed, const char* name, float scale, float offset, int64_t n, uint16_t* out) {
  if (!name || !out) return fail(LNB_EINVAL, "NULL argument");
  const uint64_t s = seed ^ fnv1a64(name);
  // counter-based generator: ranges are independent, so large tensors are filled by a few threads
  const unsigned hw = std::thread::hardware_concurrency();
  const int nt = (n < (1 << 20)) ? 1 : (int)std::min<unsigned>(16u, hw ? hw : 1u);
  if (nt <= 1) {
    synth_fill_range(s, scale, offset, 0, n, out);
    return 0;
  }
  std::vector<std::thread> th;
  const int64_t step = (n + nt - 1) / nt;
  for (int t = 0; t < nt; t++) {
    const int64_t a = (int64_t)t * step, b = std::min<int64_t>(n, a + step);
    if (a < b) th.emplace_back(synth_fill_range, s, scale, offset, a, b, out);
  }
  for (auto& x : th) x.join();
  return 0;
}
extern "C" int lnb_model_init_synthetic(lnb_model* m, uint64_t seed) {
  if (!m) return fail(LNB_EINVAL, "model is NULL");
  if (m->finalized) return fail(LNB_ESTATE, "model is finalized");
  CU(cudaSetDevice(m->device));
  static const char* lnames[9] = {"attention_norm.weight", "attention.wq.weight", "attention.wk.weight",
                                  "attention.wv.weight",   "attention.wo.weight", "ffn_norm.weight",
                                  "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight"};
  auto fill = [&](const char* name, int kind, int layer) -> int {
    int64_t rows, cols;
    full_shape(m, kind, &rows, &cols);
    const int64_t ld = (cols == 1) ? rows : cols;
    Placement p = placement(m, kind, layer);
    float scale, offset;
    synth_spec_kind(m->a, kind, &scale, &offset);
    synth_fill_kernel<<<m->sm_count * 8, 256>>>(seed ^ fnv1a64(name), scale, offset, ld, p.row0, p.col0, p.rows, p.cols,
                                                p.dst, p.panel_major ? 1 : 0, p.dpanel0, p.dpanel_stride);
    CU(cudaGetLastError());
    mark_present(m, kind, layer);
    return 0;
  };
  int rc;
  if ((rc = fill("tok_embeddings.weight", T_EMBD, -1))) return rc;
  if ((rc = fill("norm.weight", T_NORM, -1))) return rc;
  if ((rc = fill("output.weight", T_OUTPUT, -1))) return rc;
  char name[128];
  for (int l = 0; l < m->a.n_layers; l++)
    for (int k = 0; k < 9; k++) {
      snprintf(name, sizeof(name), "layers.%d.%s", l, lnames[k]);
      if ((rc = fill(name, k, l))) return rc;
    }
  CU(cudaDeviceSynchronize());
  return 0;
}

// The synthetic checkpoint as a file the UNMODIFIED reference loader can read (SURVEY 8d "Synthetic weights":
// "same bytes feed oracle, GPU path and (if ever available) the Go binary via a .pth writer").  Tensor order
// follows Meta's consolidated.00.pth (tok_embeddings, layers.*, norm, output); host-only, no CUDA call.
extern "C" int lnb_pth_write_synthetic(const char* path, const lnb_model_args* args, uint64_t seed) {
  if (!path || !args) return fail(LNB_EINVAL, "NULL argument");
  const lnb_model_args& a = *args;
  if (a.dim <= 0 || a.n_layers <= 0 || a.n_heads <= 0 || a.n_kv_heads <= 0 || a.head_dim <= 0 || a.ffn_dim <= 0 || a.vocab_size <= 0)
    return fail(LNB_EINVAL, "non-positive model dimension");
  lnb_model tmp;
  tmp.a = a;
  tmp.q_dim = a.n_heads * a.head_dim;
  tmp.kv_dim = a.n_kv_heads * a.head_dim;
  lnb::PthWriter w;
  std::string err;
  if (!w.open(path, err)) return fail(LNB_EINVAL, "%s", err.c_str());
  std::vector<uint16_t> buf;
  auto emit = [&](const char* name, int kind) -> int {
    int64_t rows, cols;
    full_shape(&tmp, kind, &rows, &cols);
    float scale, offset;
    synth_spec_kind(a, kind, &scale, &offset);
    buf.resize((size_t)(rows * cols));
    int rc = lnb_synth_fill_host(seed, name, scale, offset, rows * cols, buf.data());
    if (rc) return rc;
    std::vector<int64_t> shape;
    shape.push_back(rows);
    if (cols != 1) shape.push_back(cols);
    if (!w.add(name, lnb::PTH_BF16, buf.data(), shape, err)) return fail(LNB_EINVAL, "%s", err.c_str());
    return 0;
  };
  static const char* lnames[9] = {"attention_norm.weight", "attention.wq.weight", "attention.wk.weight",
                                  "attention.wv.weight",   "attention.wo.weight", "ffn_norm.weight",
                                  "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight"};
  int rc;
  if ((rc = emit("tok_embeddings.weight", T_EMBD))) return rc;
  char name[128];
  for (int l = 0; l < a.n_layers; l++)
    for (int k = 0; k < 9; k++) {
      snprintf(name, sizeof(name), "layers.%d.%s", l, lnames[k]);
      if ((rc = emit(name, k))) return rc;
    }
  if ((rc = emit("norm.weight", T_NORM))) return rc;
  if ((rc = emit("output.weight", T_OUTPUT))) return rc;
  if (!w.finish(err)) return fail(LNB_EINVAL, "%s", err.c_str());
  return 0;
}

// ---- tables ---------------------------------------------------------------------------------
extern "C" int lnb_model_set_rope_table(lnb_model* m, const float* cis, int rows) {
  if (!m || !cis || rows <= 0) return fail(LNB_EINVAL, "bad argument");
  if (m->finalized) return fail(LNB_ESTATE, "model is finalized");
  CU(cudaSetDevice(m->device));
  cudaFree(m->cis);
  m->cis = nullptr;
  const size_t bytes = (size_t)rows * (m->a.head_dim / 2) * 2 * sizeof(float);
  CU(cudaMalloc((void**)&m->cis, bytes));
  CU(cudaMemcpy(m->cis, cis, bytes, cudaMemcpyHostToDevice));
  m->cis_rows = rows;
  m->cis_set = true;
  return 0;
}
extern "C" int lnb_model_set_silu_table(lnb_model* m, const uint16_t* tab) {
  if (!m || !tab) return fail(LNB_EINVAL, "bad argument");
  if (m->finalized) return fail(LNB_ESTATE, "model is finalized");
  CU(cudaSetDevice(m->device));
  CU(cudaMemcpy(m->silu_tab, tab, 65536 * 2, cudaMemcpyHostToDevice));
  m->silu_set = true;
  return 0;
}
extern "C" int lnb_model_get_rope_table(lnb_model* m, float* out, int rows) {
  if (!m || !out || !m->cis || rows > m->cis_rows) return fail(LNB_EINVAL, "bad argument / table not built");
  CU(cudaSetDevice(m->device));
  CU(cudaMemcpy(out, m->cis, (size_t)rows * (m->a.head_dim / 2) * 2 * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}
extern "C" int lnb_model_get_silu_table(lnb_model* m, uint16_t* out) {
  if (!m || !out) return fail(LNB_EINVAL, "bad argument");
  CU(cudaSetDevice(m->device));
  CU(cudaMemcpy(out, m->silu_tab, 65536 * 2, cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int lnb_model_finalize(lnb_model* m) {
  if (!m) return fail(LNB_EINVAL, "model is NULL");
  if (m->finalized) return 0;
  if (!m->have_embd) return fail(LNB_ESTATE, "missing tensor tok_embeddings.weight");
  if (!m->have_norm) return fail(LNB_ESTATE, "missing tensor norm.weight");
  if (!m->have_output) return fail(LNB_ESTATE, "missing tensor output.weight");
  for (int l = 0; l < m->a.n_layers; l++)
    if (m->layers[l].have != 0x1ffu) return fail(LNB_ESTATE, "layer %d: missing tensors (mask 0x%x)", l, m->layers[l].have);
  CU(cudaSetDevice(m->device));
  if (!m->cis_set) {
    std::vector<float> cis;
    const int rows = m->a.max_seq_len * 2;  // llamatransformer.go:109
    build_rope_table(m->a.head_dim, rows, m->a.rope_theta, m->a.use_scaled_rope != 0, cis);
    int rc = lnb_model_set_rope_table(m, cis.data(), rows);
    if (rc) return rc;
  }
  if (!m->silu_set) {
    std::vector<uint16_t> tab;
    build_silu_table(tab);
    int rc = lnb_model_set_silu_table(m, tab.data());
    if (rc) return rc;
  }
  if (m->staging) { cudaFree(m->staging); m->staging = nullptr; m->staging_bytes = 0; }
  CU(cudaDeviceSynchronize());
  m->finalized = true;
  return 0;
}

// ------------------------------------------------------------------------------------------
// GEMV dispatch
// LNB_ACC_STRICT, one activation row.  The accumulation chain is issue-bound on its scheduler
// (~2.4 instructions per k at one instruction per 2 cycles), so every chain warp needs an SMSP to
// itself: ONE CTA per SM (>113 KB of shared memory each) holding 1, 2 or 4 chain warps (warps 1..4
// sit on SMSPs 1,2,3,0; the producer warp 0 sleeps on its mbarrier), picked from N so that the grid
// stays close to one wave.  Two chain warps on one scheduler run at half speed each.
using CfgS1 = GemvCfg<32, 1, 1, 512, 3>;    // N <= 32*kWaveSMs rows
using CfgS1M = GemvCfg<64, 1, 1, 512, 3>;   // N <= 64*kWaveSMs
using CfgS1W = GemvCfg<128, 1, 1, 256, 3>;  // larger N (w1|w3, LM head): several waves, HBM-bound
using CfgS2 = GemvCfg<32, 1, 2, 256, 4>;
using CfgS8 = GemvCfg<32, 1, 8, 256, 4>;
using CfgF1 = GemvCfg<32, 8, 1, 256, 4>;
using CfgF1L = GemvCfg<32, 8, 1, 512, 3>;  // at most one CTA per SM (wo, w2): larger bulk copies
using CfgF2 = GemvCfg<32, 8, 2, 256, 4>;
using CfgF8 = GemvCfg<32, 8, 8, 256, 4>;

static const size_t kMaxSmem = 227 * 1024;
static const int kWaveSMs = 132;   // H100 SXM: one wave of one-CTA-per-SM GEMV blocks

// LAUNCH_PDL: programmatic stream serialization -- the kernel may start while its predecessor drains and waits for it in
// pdl_wait().  LAUNCH_COOP: all CTAs co-resident (they wait for each other), or the launch fails.
enum LaunchAttr { LAUNCH_PLAIN, LAUNCH_PDL, LAUNCH_COOP };
struct Launcher {
  cudaStream_t stream;
  LaunchAttr attr;
  int64_t* counter;   // the session's launch count, or NULL
};

template <typename... Args>
static int launch_kernel(const Launcher& L, void (*kern)(Args...), dim3 grid, dim3 block, size_t smem, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = L.stream;
  cudaLaunchAttribute at[1];
  if (L.attr == LAUNCH_COOP) {
    at[0].id = cudaLaunchAttributeCooperative;
    at[0].val.cooperative = 1;
  } else {
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
  }
  cfg.attrs = at;
  cfg.numAttrs = L.attr == LAUNCH_PLAIN ? 0 : 1;
  CU(cudaLaunchKernelEx(&cfg, kern, args...));
  if (L.counter) (*L.counter)++;
  return 0;
}

// The opt-in to large dynamic shared memory is per kernel AND per device (context): one mask of devices per kernel,
// which is why the kernel itself is the template argument.
template <auto Kern>
static int smem_opt_in(int bytes) {
  static std::atomic<uint64_t> done{0};
  int dev = 0;
  CU(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(done.load(std::memory_order_relaxed) & bit)) {
    CU(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    done.fetch_or(bit, std::memory_order_relaxed);
  }
  return 0;
}

// ---- streamed attention (sdpa_stream.cuh) ---------------------------------------------------------------------
// Scratch of one launch group of `rows` rows over keys [0, t_stride): bf16 scores, FAST chunk row sums and chunk
// outputs.  The rows of a call are processed in groups of `rows`, so the score scratch stays within kSsScoreBudget
// however many rows a prompt has.
static const size_t kSsScoreBudget = (size_t)64 << 20;
struct SsScratch {
  uint16_t* sc = nullptr;
  double* z = nullptr;
  float* op = nullptr;
  int rows = 0, t_stride = 0, n_chunks = 0;
};
static bool ss_shape_ok(int hd, int n_rep) { return hd % 8 == 0 && hd <= 128 && n_rep >= 1 && n_rep <= 8; }
// sizes for keys [0, T) and at most max_rows rows per call (bytes per buffer)
static void ss_plan(SsScratch& x, int T, int max_rows, int n_heads, int hd, size_t* sc_b, size_t* z_b, size_t* op_b) {
  x.t_stride = (T + SS_VT - 1) / SS_VT * SS_VT;
  x.n_chunks = (x.t_stride + SS_CH - 1) / SS_CH;
  const size_t row = (size_t)n_heads * x.t_stride * 2;
  x.rows = (int)std::max<size_t>(1, std::min<size_t>({kSsScoreBudget / row, (size_t)max_rows, (size_t)65535}));
  *sc_b = (size_t)x.rows * row;
  *z_b = (size_t)x.rows * n_heads * x.n_chunks * 8;
  *op_b = (size_t)x.rows * n_heads * x.n_chunks * hd * 4;
}
// STRICT output chains: the d-range of one CTA (more CTAs per KV head; each chain still runs t = 0..p in order)
static int ss_dsplit(int hd) { return hd % 32 == 0 ? 4 : hd % 16 == 0 ? 2 : 1; }
// all `rows` rows of P (P.q, P.out, positions and caches set by the caller)
static int launch_stream_attn(const Launcher& L, StreamAttn P, int rows, int n_kv, const SsScratch& x) {
  const int dsplit = P.strict ? ss_dsplit(P.hd) : 1;
  const size_t s_scores = ss_scores_smem(P.hd, P.n_rep), s_out = ss_out_smem(P.hd, P.n_rep, dsplit);
  // the largest shape ss_shape_ok admits (head_dim 128, n_rep 8, FAST); the kernel's static shared memory comes on top
  if (int rc = smem_opt_in<ss_out_kernel>((int)ss_out_smem(128, 8, 1))) return rc;
  P.sc = x.sc; P.zpart = x.z; P.opart = x.op; P.t_stride = x.t_stride; P.n_chunks = x.n_chunks;
  for (int r0 = 0; r0 < rows; r0 += x.rows) {
    const int n = std::min(x.rows, rows - r0);
    P.row0 = r0;
    int rc;
    if ((rc = launch_kernel(L, ss_scores_kernel, dim3(n_kv, n, x.n_chunks), dim3(SS_KT), s_scores, P))) return rc;
    if (P.strict) {
      if ((rc = launch_kernel(L, ss_zsum_kernel, dim3(P.n_heads, n), dim3(128), 0, P))) return rc;
      if ((rc = launch_kernel(L, ss_out_kernel, dim3(n_kv * dsplit, n), dim3(P.n_rep * P.hd / dsplit), s_out, P, dsplit))) return rc;
    } else {
      if ((rc = launch_kernel(L, ss_out_kernel, dim3(n_kv, n, x.n_chunks), dim3(P.n_rep * P.hd), s_out, P, 1))) return rc;
      if ((rc = launch_kernel(L, ss_combine_kernel, dim3(P.n_heads, n), dim3(P.hd), 0, P))) return rc;
    }
  }
  return 0;
}

template <class Cfg, int PRO, int EPI>
static int launch_gemv_cfg(const Launcher& L, const GemvParams& p) {
  if (int rc = smem_opt_in<gemv_kernel<Cfg, PRO, EPI>>((int)kMaxSmem)) return rc;
  return launch_kernel(L, gemv_kernel<Cfg, PRO, EPI>, dim3((p.N / 8 + Cfg::kP - 1) / Cfg::kP), dim3(Cfg::kThreads),
                       Cfg::smem_bytes(p.K), p);
}

// picks the row-block size: largest MB in {8,2,1} that is useful for M and whose smem fits.  mb_rows > 0 chooses it for
// that many rows instead of M_total (ragged calls pass 8: the block size, and with it a row's FAST summation order, then
// depends on K alone, not on how many rows share the call)
template <int PRO, int EPI>
static int launch_gemv(const Launcher& L, int mode, GemvParams p, int M_total, int mb_rows = 0) {
  if (p.N % 16 || p.K % 8) return fail(LNB_EINVAL, "gemv: N %d must be a multiple of 16 and K %d of 8", p.N, p.K);  // 16: panel pairs
  if ((EPI == EPI_QKV_ROPE || EPI == EPI_SWIGLU) && p.N % 32) return fail(LNB_EINVAL, "gemv: N %d must be a multiple of 32", p.N);
  const bool strict = (mode == LNB_ACC_STRICT);
  p.strict_norm = strict ? 1 : 0;
  const int mb_for = mb_rows > 0 ? mb_rows : M_total;
  int mb = 1;
  if (mb_for >= 3 && (strict ? CfgS8::smem_bytes(p.K) : CfgF8::smem_bytes(p.K)) <= kMaxSmem) mb = 8;
  else if (mb_for >= 2 && (strict ? CfgS2::smem_bytes(p.K) : CfgF2::smem_bytes(p.K)) <= kMaxSmem) mb = 2;
  if ((strict ? CfgS1::smem_bytes(p.K) : CfgF1::smem_bytes(p.K)) > kMaxSmem)
    return fail(LNB_EINVAL, "gemv: K %d too large for shared memory", p.K);
  const uint16_t* x0 = p.x;
  uint16_t* ob0 = p.out_bf16;
  float* of0 = p.out_f32;
  const uint16_t* res0 = p.res;
  const float* rs0 = p.rscale;
  const int moff0 = p.m_off;
  LnbDevState* st0 = p.st;
  const int arg_row = p.argmax_row;
  for (int m0 = 0; m0 < M_total; m0 += mb) {
    p.M = (M_total - m0 < mb) ? (M_total - m0) : mb;
    p.x = x0 + (size_t)m0 * p.ldx;
    p.out_bf16 = ob0 ? ob0 + (size_t)m0 * p.ldo : nullptr;
    p.out_f32 = of0 ? of0 + (size_t)m0 * p.ldo : nullptr;
    p.res = res0 ? res0 + (size_t)m0 * p.ldo : nullptr;
    p.rscale = rs0 ? rs0 + m0 : nullptr;
    p.m_off = moff0 + m0;
    if (EPI == EPI_LOGITS) {
      const bool covers = st0 && arg_row >= m0 && arg_row < m0 + p.M;
      p.st = covers ? st0 : nullptr;
      p.argmax_row = covers ? arg_row - m0 : -1;
    }
    int rc;
    if (strict) {
      if (mb == 1 && p.N > 64 * kWaveSMs && p.N % 128 == 0 && CfgS1W::smem_bytes(p.K) <= kMaxSmem) rc = launch_gemv_cfg<CfgS1W, PRO, EPI>(L, p);
      else if (mb == 1 && p.N > 32 * kWaveSMs && p.N % 64 == 0 && CfgS1M::smem_bytes(p.K) <= kMaxSmem) rc = launch_gemv_cfg<CfgS1M, PRO, EPI>(L, p);
      else if (mb == 1) rc = launch_gemv_cfg<CfgS1, PRO, EPI>(L, p);
      else if (mb == 8) rc = launch_gemv_cfg<CfgS8, PRO, EPI>(L, p);
      else rc = launch_gemv_cfg<CfgS2, PRO, EPI>(L, p);
    } else {
      if (mb == 8) rc = launch_gemv_cfg<CfgF8, PRO, EPI>(L, p);
      else if (mb == 2) rc = launch_gemv_cfg<CfgF2, PRO, EPI>(L, p);
      else if (p.N <= 32 * kWaveSMs && CfgF1L::smem_bytes(p.K) <= kMaxSmem) rc = launch_gemv_cfg<CfgF1L, PRO, EPI>(L, p);
      else rc = launch_gemv_cfg<CfgF1, PRO, EPI>(L, p);
    }
    if (rc) return rc;
  }
  return 0;
}

// LNB_ACC_STRICT RMSNorm scale r[row] (the reference's sequential fp32 sum of squares, bit-exact).  Three
// interchangeable kernels, identical bits: 1 = one-thread FADD chain (rms_scale_kernel), 2 = iterative binade
// scan, 3 = one-pass predict / fold / walk (both seqsum.cuh; need a row length that fits seq_scan_shape).
// algo 0 = the model path's choice: LNB_RMS_ALGO=chain|scan|seg, else kRmsDefaultAlgo.
enum { RMS_AUTO = 0, RMS_CHAIN = 1, RMS_SCAN = 2, RMS_SEG = 3, RMS_ENGINE = 4 };   // 4 = the decode engine's in-CTA variant (engine.cuh)
static const int kRmsDefaultAlgo = RMS_SEG;  // the fewest dependent steps of the three
static int rms_default_algo() {
  static const int a = [] {
    const char* e = getenv("LNB_RMS_ALGO");
    if (e && !strcmp(e, "chain")) return (int)RMS_CHAIN;
    if (e && !strcmp(e, "scan")) return (int)RMS_SCAN;
    if (e && !strcmp(e, "seg")) return (int)RMS_SEG;
    return kRmsDefaultAlgo;
  }();
  return a;
}
static int launch_rms_scale(const Launcher& L, const uint16_t* x, int ldx, float* r, int rows, int D, float eps, int algo = RMS_AUTO) {
  int ch = 0, nt = 0;
  if (algo == RMS_AUTO) algo = rms_default_algo();
  if (algo != RMS_CHAIN && !seq_scan_shape(D, &ch, &nt)) algo = RMS_CHAIN;
  if (algo == RMS_SCAN) {
    switch (ch) {
      case 2: return launch_kernel(L, rms_scale_scan_kernel<2>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
      case 4: return launch_kernel(L, rms_scale_scan_kernel<4>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
      case 8: return launch_kernel(L, rms_scale_scan_kernel<8>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
      default: return launch_kernel(L, rms_scale_scan_kernel<16>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
    }
  }
  if (algo == RMS_SEG) {
    switch (ch) {
      case 2: return launch_kernel(L, rms_scale_seg_kernel<2>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
      case 4: return launch_kernel(L, rms_scale_seg_kernel<4>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
      case 8: return launch_kernel(L, rms_scale_seg_kernel<8>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
      default: return launch_kernel(L, rms_scale_seg_kernel<16>, dim3(rows), dim3(nt), 0, x, ldx, r, D, eps);
    }
  }
  return launch_kernel(L, rms_scale_kernel, dim3(rows), dim3(128), (size_t)D * 4, x, ldx, r, D, eps);
}

// tensor-core GEMM launcher (prefill): grid = (N/128, ceil(M/128))
template <int EPI>
static int launch_gemm_tc(const Launcher& L, const GemmTcParams& p) {
  if (p.N % TC_BN || p.K % TC_KT) return fail(LNB_EINVAL, "gemm_tc: N %d and K %d must be multiples of 128", p.N, p.K);
  if (int rc = smem_opt_in<gemm_tc_kernel<EPI>>(TC_SMEM)) return rc;
  return launch_kernel(L, gemm_tc_kernel<EPI>, dim3((p.M + TC_BM - 1) / TC_BM, p.N / TC_BN), dim3(TC_THREADS), TC_SMEM, p);
}
static bool tc_eligible(int M, int N, int K) { return M >= 32 && N % TC_BN == 0 && K % TC_KT == 0; }

// ------------------------------------------------------------------------------------------
// session
__global__ void set_state_kernel(LnbDevState* st, int pos, int n_rows, int next_token, int reset_step) {
  st->pos = pos;
  st->safe_rows = pos;  // rows before this call's first position come from earlier, synchronised calls
  st->n_rows = n_rows;
  st->amax_key = LNB_ARGMAX_EMPTY;
  st->done_ctr = 0;
  if (next_token >= 0) st->next_token = next_token;
  if (reset_step) st->step = 0;
}
__global__ void set_p2p_epoch_kernel(LnbDevState* st, uint32_t e) {
  st->ar_epoch = e;
  st->ar_error = 0;
  st->ar_done2 = 0;
}
// tensor-parallel tail of the LM head: decode the reduced key, advance the decode state
__global__ void publish_kernel(LnbDevState* st, int advance, int32_t* tok_out) {
  pdl_launch_dependents();
  pdl_wait();
  const unsigned long long key = st->amax_key;
  const int32_t tok = (key == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull));
  st->next_token = tok;
  st->amax_key = LNB_ARGMAX_EMPTY;
  st->done_ctr = 0;
  if (advance) {
    if (tok_out) tok_out[st->step] = tok;
    st->step += 1;
    st->pos += 1;
  }
}

// words of a ragged call's row map [tokens | row_seq | row_pos | last row of each segment]: `rows` words each, <= 8 segments
static size_t row_map_words(int max_rows) { return (size_t)max_rows * 3 + 8; }

struct lnb_session {
  lnb_model* m = nullptr;
  int seq_len = 0, max_rows = 1, mode = LNB_ACC_FAST;
  cudaStream_t stream = nullptr;
  uint16_t *x = nullptr, *h1 = nullptr, *q = nullptr, *o = nullptr, *mbuf = nullptr;
  float* part = nullptr;
  float* rs = nullptr;  // [max_rows] strict-mode RMSNorm scales
  // tensor-core prefill path (LNB_ACC_FAST, S >= 32): X8-layout activations + raw GEMM outputs
  uint16_t *xn8 = nullptr, *o8 = nullptr, *m8 = nullptr, *qkv_raw = nullptr, *gu = nullptr;
  int mpad = 0;
  // peer-memory all-reduce (tp_size > 1, optional): own region + the peers' mapped regions
  uint8_t* p2p_region = nullptr;
  size_t p2p_bytes = 0;
  void* p2p_peer[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  LnbP2P p2p{};
  bool p2p_ready = false;
  float* logits = nullptr;
  size_t logits_rows = 0;
  float* logits_full = nullptr;  // tp>1: gathered [rows, vocab]
  std::vector<uint16_t*> ck, cv;
  int32_t* d_tokens = nullptr;
  LnbDevState* st = nullptr;
  int32_t* d_tok_out = nullptr;
  // pinned staging, one allocation (at h_tok) carved into three views: token ids on their way to d_tokens, or a ragged
  // call's row map on its way to d_rag [row_map_words]; the positions of a batched step on their way to d_pos_arr [8]; the
  // tokens a call hands back [seq_len + 8]
  int32_t *h_tok = nullptr, *h_pos = nullptr, *h_out = nullptr;
  uint32_t* h_err = nullptr;     // pinned mirror of st->ar_error (peer all-reduce timeout flag)
  // logits of the last forward stay in HBM (lnb_forward_device); the host reads rows / argmaxes on demand
  int kept_rows = 0;             // rows of s->logits that belong to the last forward (0: none)
  int32_t kept_last_token = -1;  // greedy token of the last kept row (fused argmax of the LM-head kernel)
  int64_t generation = 0;        // forward calls so far (a logits handle is valid for one generation)
  float* h_logits_pin = nullptr; // pinned staging for logits read-backs
  size_t h_logits_bytes = 0;
  unsigned long long* d_keys = nullptr;  // [max_rows] per-row argmax keys (tensor-parallel on-demand argmax)
  int layer_limit = 0;
  bool allow_chunked = false;    // S > 1 at startPos > 0 (chunked prefill, an extension the reference cannot express)
  // batched decode (BASELINE config 5): n_seq independent sequences share the weights; caches are
  // [n_seq][seq_len][kv]; single-sequence calls address the cache of `active_seq`
  int n_seq = 1, active_seq = 0;
  int32_t* d_pos_arr = nullptr;   // [n_seq] positions of the current batched step
  int32_t* d_next_arr = nullptr;  // [n_seq] greedy tokens of the current batched step
  bool sdpa_smem_decode = false;  // the whole K/V history of one KV head fits in shared memory
  size_t sdpa_decode_smem = 0;
  // streamed attention (sdpa_stream.cuh): every row of the session runs it when sdpa_kernel cannot hold seq_len keys
  // (stream_attn); batched steps run it when sdpa_decode_kernel cannot.  Scratch for ss.rows rows per launch group.
  bool stream_attn = false;
  SsScratch ss{};
  int32_t* d_rag = nullptr;       // the row map of a ragged call, allocated by the first one (ONE host-to-device copy per call)
  int64_t launches = 0;
  // persistent decode engine (engine.cuh): the phase list of one S=1 step in device memory
  EnginePhase* d_phases = nullptr;
  int n_phases = 0, phases_cap = 0;
  unsigned int* d_bar = nullptr;
  // tagged activation vectors of the engine ({tag:16 | bf16:16} words): residual stream x, post-attention stream h1,
  // q|k|v of the step, attention output o, FFN hidden m
  uint32_t *x_t = nullptr, *h1_t = nullptr, *qkv_t = nullptr, *o_t = nullptr, *m_t = nullptr;
  // batch engine (engine_batch.cuh): chunk-major bf16 activations [K/8][8][8] of up to 8 sequences, its phase list, argmax keys
  uint16_t *bx = nullptr, *bh1 = nullptr, *bq = nullptr, *bo = nullptr, *bm = nullptr, *bxn = nullptr;
  int batch_tc = 0;     // FAST batch engine: projections on the tensor cores (batch_engine_kernel<0>)
  BatchPhase* d_bphases = nullptr;
  int n_bphases = 0;
  unsigned long long* d_bkeys = nullptr;
  int bkey_layers = -1;
  const float* bkey_logits = nullptr;
  uint32_t eng_tag = 1;          // next free tag (tags of one launch: [eng_tag, eng_tag + n_steps * n_phases))
  bool last_was_engine = false;  // the residual stream of the last forward lives in x_t
  unsigned long long* d_prof = nullptr;   // LNB_ENGINE_PROF=1: per-CTA cycle counters of the engine's consumer thread 0
  int eng_state = 0;             // 0 = not probed, 1 = usable, -1 = this session uses the kernel chain
  bool eng_single_default = true; // single-sequence S=1 steps use the engine (false: single-GPU FAST, where the kernel chain is faster)
  std::string eng_why;           // why not
  int eng_key_seq = -1, eng_key_layers = -1, eng_key_kind = -2;
  const float* eng_key_logits = nullptr;
  cudaGraphExec_t graph = nullptr;
  int64_t graph_launches = 0;    // kernels one replay of `graph` launches (counted while it was captured)
  bool graph_tried = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::mutex mu;
  // seeded sampling (sample.cuh, lnb_session_set_sampling), allocated by the first sampler set: the parameters of each
  // sequence in device memory (a captured graph reads them there), the weights of up to n_seq rows, the sampled token of
  // a single-sequence forward (st->next_token keeps the greedy one)
  lnb_sampling* d_samp = nullptr;           // [n_seq]
  unsigned long long* d_samp_w = nullptr;   // [samp_rows][vocab]
  unsigned long long* d_samp_cand = nullptr;   // [samp_rows][SMP_MERGE] split-sampler candidates, then [samp_rows] u32 counters
  int samp_rows = 0;                        // rows one sampler launch may draw: n_seq, grown by speculative calls (samp_grow)
  int32_t* d_samp_tok = nullptr;
  bool samp_on[8] = {false, false, false, false, false, false, false, false};
  bool graph_sampled = false;               // the captured decode graph ends in the sampler ...
  const float* graph_logits = nullptr;      // ... which reads this logits buffer
  // token log-probabilities (logprob.cuh, lnb_session_set_logprobs), allocated by the first enable: the records of every
  // sequence and position, the top_n of each sequence in device memory (a captured graph reads it there), the row table
  // and scratch of one job of up to lp_rows rows, and the targets of lnb_score
  LpRecord* d_lp_rec = nullptr;             // [n_seq][seq_len + 1], keyed by the position of the scored token
  int32_t* d_lp_top = nullptr;              // [n_seq]
  int32_t* d_lp_tgt = nullptr;              // [max_rows]
  LpRow* d_lp_rows = nullptr;               // [lp_rows]
  LpRow* h_lp_rows = nullptr;               // pinned staging of d_lp_rows
  unsigned long long* d_lp_cand = nullptr;  // [lp_rows][slices][LP_TOP], then [lp_rows][slices] + [lp_rows] u32 counters
  int lp_rows = 0;
  int lp_top[8] = {-1, -1, -1, -1, -1, -1, -1, -1};   // -1: logprobs off
  bool graph_lp = false;                    // the captured decode graph ends in the logprob job
  // penalties (penalty.cuh, lnb_session_set_penalties), allocated by the first enable: the token history of every sequence
  // and position, the parameters of each sequence in device memory (a captured graph reads them there), and one job's
  // counts and processed rows
  int32_t* d_hist = nullptr;                // [n_seq][seq_len] the token fed at each position, -1: none
  lnb_penalties* d_pen = nullptr;           // [n_seq]
  unsigned int* d_pen_cnt = nullptr;        // [PEN_MAX_ROWS][vocab] (zero between jobs)
  float* d_pen_out = nullptr;               // [PEN_MAX_ROWS][vocab] l', read by the sampler
  bool pen_on[8] = {false, false, false, false, false, false, false, false};
  bool graph_pen = false, graph_greedy = false;   // the captured decode graph runs the penalty job / the greedy slot
};

// a sequence whose tokens the sampler draws (sampled, or penalized: greedy is then the sampler's rank 0 of l')
static bool processed(const lnb_session* s, int seq) { return s->samp_on[seq] || s->pen_on[seq]; }

static int set_state(lnb_session* s, int pos, int n_rows, int next_token, bool reset_step) {
  return launch_kernel(Launcher{s->stream, LAUNCH_PLAIN, &s->launches}, set_state_kernel, dim3(1), dim3(1), 0, s->st, pos, n_rows,
                       next_token, reset_step ? 1 : 0);
}
// layers a forward runs (lnb_session_set_layer_limit; <= 0: all)
static int active_layers(const lnb_session* s) {
  const int n = s->m->a.n_layers;
  return (s->layer_limit > 0 && s->layer_limit < n) ? s->layer_limit : n;
}
// budget of one in-kernel wait for a peer (a late or dead rank yields LNB_ETIMEOUT instead of a hung GPU):
// LNB_P2P_TIMEOUT_MS, default 1500; <= 0 waits forever (0 ns)
static unsigned long long p2p_timeout_ns() {
  const char* e = getenv("LNB_P2P_TIMEOUT_MS");
  const long ms = e ? atol(e) : 1500;
  return ms > 0 ? (unsigned long long)ms * 1000000ull : 0ull;
}

static int session_create_impl(lnb_model* m, int seq_len, int max_rows, int acc_mode, int n_seq, lnb_session** out);
extern "C" int lnb_session_create(lnb_model* m, int seq_len, int max_rows, int acc_mode, lnb_session** out) {
  return session_create_impl(m, seq_len, max_rows, acc_mode, 1, out);
}
extern "C" int lnb_session_create_batch(lnb_model* m, int seq_len, int n_seq, int max_rows, int acc_mode, lnb_session** out) {
  if (n_seq < 1 || n_seq > 8) return fail(LNB_EINVAL, "n_seq must be 1..8");
  return session_create_impl(m, seq_len, max_rows < n_seq ? n_seq : max_rows, acc_mode, n_seq, out);
}
static int session_create_impl(lnb_model* m, int seq_len, int max_rows, int acc_mode, int n_seq, lnb_session** out) {
  if (!m || !out) return fail(LNB_EINVAL, "NULL argument");
  if (!m->finalized) return fail(LNB_ESTATE, "model is not finalized");
  if (seq_len <= 0 || max_rows <= 0) return fail(LNB_EINVAL, "seq_len and max_rows must be positive");
  if (seq_len > m->cis_rows) return fail(LNB_EINVAL, "seq_len %d exceeds the RoPE table (%d rows)", seq_len, m->cis_rows);
  if (acc_mode != LNB_ACC_STRICT && acc_mode != LNB_ACC_FAST) return fail(LNB_EINVAL, "bad acc_mode %d", acc_mode);
  // sdpa_kernel holds a row's seq_len scores in shared memory; beyond that every row of the session streams
  const bool stream_attn = (size_t)seq_len * 12 + (size_t)m->a.head_dim * 4 > 200 * 1024;
  if (stream_attn && !ss_shape_ok(m->a.head_dim, m->a.n_heads / m->a.n_kv_heads))
    return fail(LNB_EINVAL, "seq_len %d needs the streamed attention kernel, which serves head_dim <= 128 and n_rep <= 8", seq_len);
  CU(cudaSetDevice(m->device));
  CU(cudaFuncSetAttribute(sdpa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  CU(cudaFuncSetAttribute(sdpa_prefill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_SMEM));
  CU(cudaFuncSetAttribute(sdpa_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ST_SMEM));
  lnb_session* s = new lnb_session();
  s->m = m;
  s->seq_len = seq_len;
  s->max_rows = max_rows;
  s->mode = acc_mode;
  s->n_seq = n_seq;
  const lnb_model_args& a = m->a;
  {
    const int n_rep = a.n_heads / a.n_kv_heads;
    const size_t need = (size_t)seq_len * ((a.head_dim + 8) + a.head_dim) * 2 + (size_t)n_rep * ((size_t)a.head_dim * 4 + (size_t)seq_len * 12 + 5 * 8) + 256;
    if (need <= 200 * 1024 && n_rep <= 8 && a.head_dim <= 128 && a.head_dim % 8 == 0) {
      s->sdpa_smem_decode = true;
      s->sdpa_decode_smem = need;
      CU(cudaFuncSetAttribute(sdpa_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
  }
  s->stream_attn = stream_attn;
  cudaError_t e = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
  // every allocation is counted, so a failure can say how much the session asked for
  size_t asked = 0, failed_bytes = 0;
  auto al = [&](void** p, size_t bytes) {
    asked += bytes;
    if (e != cudaSuccess) return;
    e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) { failed_bytes = bytes; *p = nullptr; }
  };
  if (stream_attn || (!s->sdpa_smem_decode && ss_shape_ok(a.head_dim, a.n_heads / a.n_kv_heads))) {
    // streamed rows: every row of a long session, or the n_seq rows of a batched step
    size_t sc_b, z_b, op_b;
    ss_plan(s->ss, seq_len, stream_attn ? max_rows : n_seq, m->q_l / a.head_dim, a.head_dim, &sc_b, &z_b, &op_b);
    al((void**)&s->ss.sc, sc_b);
    al((void**)&s->ss.z, z_b);
    al((void**)&s->ss.op, op_b);
  }
  al((void**)&s->x, (size_t)max_rows * a.dim * 2);
  al((void**)&s->h1, (size_t)max_rows * a.dim * 2);
  al((void**)&s->q, (size_t)max_rows * m->q_l * 2);
  al((void**)&s->o, (size_t)max_rows * m->q_l * 2);
  al((void**)&s->mbuf, (size_t)max_rows * m->ffn_l * 2);
  al((void**)&s->part, (size_t)max_rows * a.dim * 4);
  al((void**)&s->rs, (size_t)max_rows * 4);
  if (max_rows >= 32 && acc_mode == LNB_ACC_FAST) {
    s->mpad = (max_rows + TC_BM - 1) / TC_BM * TC_BM;
    al((void**)&s->xn8, (size_t)s->mpad * a.dim * 2);
    al((void**)&s->o8, (size_t)s->mpad * m->q_l * 2);
    al((void**)&s->m8, (size_t)s->mpad * m->ffn_l * 2);
    al((void**)&s->qkv_raw, (size_t)max_rows * (m->q_l + 2 * m->kv_l) * 2);
    al((void**)&s->gu, (size_t)max_rows * 2 * m->ffn_l * 2);
  }
  al((void**)&s->d_tokens, (size_t)max_rows * 4);
  al((void**)&s->st, sizeof(LnbDevState));
  al((void**)&s->d_tok_out, (size_t)seq_len * 4);
  s->ck.assign(a.n_layers, nullptr);
  s->cv.assign(a.n_layers, nullptr);
  const size_t cbytes = (size_t)n_seq * seq_len * m->kv_l * 2;
  al((void**)&s->d_pos_arr, 8 * 4);
  al((void**)&s->d_next_arr, 8 * 4);
  for (int l = 0; l < a.n_layers; l++) {
    al((void**)&s->ck[l], cbytes);
    al((void**)&s->cv[l], cbytes);
    if (e == cudaSuccess) e = cudaMemsetAsync(s->ck[l], 0, cbytes, s->stream);  // ml.Zeros, inferencecontext.go:31-43
    if (e == cudaSuccess) e = cudaMemsetAsync(s->cv[l], 0, cbytes, s->stream);
  }
  if (e == cudaSuccess) e = cudaMemsetAsync(s->st, 0, sizeof(LnbDevState), s->stream);
  const size_t in_words = row_map_words(max_rows);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&s->h_tok, (in_words + 8 + seq_len + 8) * 4);
  if (e == cudaSuccess) { s->h_pos = s->h_tok + in_words; s->h_out = s->h_tok + in_words + 8; }
  if (e == cudaSuccess) e = cudaMallocHost((void**)&s->h_err, 64);
  if (e == cudaSuccess) *s->h_err = 0;
  if (e == cudaSuccess) e = cudaEventCreate(&s->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&s->ev1);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s->stream);
  if (e != cudaSuccess) {
    cudaGetLastError();
    lnb_session_destroy(s);
    cudaGetLastError();
    return fail(LNB_ENOMEM, "session allocation failed: %zu bytes of device memory asked for (KV cache %zu bytes), %zu-byte allocation: %s",
                asked, (size_t)2 * a.n_layers * cbytes, failed_bytes, cudaGetErrorString(e));
  }
  *out = s;
  return 0;
}

extern "C" int lnb_session_destroy(lnb_session* s) {
  if (!s) return 0;
  cudaSetDevice(s->m->device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  if (s->graph) cudaGraphExecDestroy(s->graph);
  cudaFree(s->x); cudaFree(s->h1); cudaFree(s->q); cudaFree(s->o); cudaFree(s->mbuf); cudaFree(s->part); cudaFree(s->rs);
  cudaFree(s->xn8); cudaFree(s->o8); cudaFree(s->m8); cudaFree(s->qkv_raw); cudaFree(s->gu);
  for (int r = 0; r < 8; r++)
    if (s->p2p_peer[r]) cudaIpcCloseMemHandle(s->p2p_peer[r]);
  cudaFree(s->p2p_region);
  cudaFree(s->d_phases); cudaFree(s->d_bar); cudaFree(s->d_prof);
  cudaFree(s->x_t); cudaFree(s->h1_t); cudaFree(s->qkv_t); cudaFree(s->o_t); cudaFree(s->m_t);
  cudaFree(s->bx); cudaFree(s->bh1); cudaFree(s->bq); cudaFree(s->bo); cudaFree(s->bm); cudaFree(s->bxn); cudaFree(s->d_bphases); cudaFree(s->d_bkeys);
  cudaFree(s->logits); cudaFree(s->logits_full); cudaFree(s->d_tokens); cudaFree(s->st); cudaFree(s->d_tok_out); cudaFree(s->d_pos_arr); cudaFree(s->d_next_arr);
  cudaFree(s->ss.sc); cudaFree(s->ss.z); cudaFree(s->ss.op);
  cudaFree(s->d_rag);
  cudaFree(s->d_samp); cudaFree(s->d_samp_w); cudaFree(s->d_samp_tok); cudaFree(s->d_samp_cand);
  cudaFree(s->d_lp_rec); cudaFree(s->d_lp_top); cudaFree(s->d_lp_tgt); cudaFree(s->d_lp_rows); cudaFree(s->d_lp_cand);
  if (s->h_lp_rows) cudaFreeHost(s->h_lp_rows);
  cudaFree(s->d_hist); cudaFree(s->d_pen); cudaFree(s->d_pen_cnt); cudaFree(s->d_pen_out);
  for (auto p : s->ck) cudaFree(p);
  for (auto p : s->cv) cudaFree(p);
  if (s->h_tok) cudaFreeHost(s->h_tok);
  if (s->h_err) cudaFreeHost(s->h_err);
  if (s->h_logits_pin) cudaFreeHost(s->h_logits_pin);
  cudaFree(s->d_keys);
  if (s->ev0) cudaEventDestroy(s->ev0);
  if (s->ev1) cudaEventDestroy(s->ev1);
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
  return 0;
}

// Peer-memory all-reduce setup.  Step 1 on every rank: export (allocates this session's region and
// returns its 64-byte CUDA IPC handle).  The host gathers the tp_size handles (any channel).  Step 2 on
// every rank: import all handles (index = rank).  From then on the decode path of this session pushes
// its Wo / w2 partials and argmax keys straight into the peers' memory instead of calling NCCL.
extern "C" int lnb_session_p2p_export(lnb_session* s, void* handle64) {
  if (!s || !handle64) return fail(LNB_EINVAL, "NULL argument");
  lnb_model* m = s->m;
  if (m->tp_size < 2 || m->tp_size > 8) return fail(LNB_EINVAL, "peer all-reduce needs 2..8 ranks");
  CU(cudaSetDevice(m->device));
  if (!s->p2p_region) {
    const size_t slot = (size_t)s->max_rows * m->a.dim;
    s->p2p_bytes = (size_t)2 * m->tp_size * slot * sizeof(uint2);
    CU(cudaMalloc((void**)&s->p2p_region, s->p2p_bytes));
    CU(cudaMemset(s->p2p_region, 0, s->p2p_bytes));
    CU(cudaDeviceSynchronize());
  }
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, s->p2p_region));
  static_assert(sizeof(h) == 64, "CUDA IPC handle size");
  memcpy(handle64, &h, 64);
  return 0;
}
extern "C" int lnb_session_p2p_import(lnb_session* s, const void* handles, int n) {
  if (!s || !handles) return fail(LNB_EINVAL, "NULL argument");
  lnb_model* m = s->m;
  if (n != m->tp_size) return fail(LNB_EINVAL, "expected %d handles, got %d", m->tp_size, n);
  if (!s->p2p_region) return fail(LNB_ESTATE, "call lnb_session_p2p_export first");
  CU(cudaSetDevice(m->device));
  std::lock_guard<std::mutex> lk(s->mu);
  for (int r = 0; r < n; r++) {
    uint8_t* base;
    if (r == m->tp_rank) {
      base = s->p2p_region;
    } else {
      cudaIpcMemHandle_t h;
      memcpy(&h, (const uint8_t*)handles + (size_t)r * 64, 64);
      void* q = nullptr;
      CU(cudaIpcOpenMemHandle(&q, h, cudaIpcMemLazyEnablePeerAccess));
      s->p2p_peer[r] = q;
      base = (uint8_t*)q;
    }
    s->p2p.data[r] = reinterpret_cast<uint2*>(base);
  }
  s->p2p.rank = m->tp_rank;
  s->p2p.n = n;
  s->p2p.slot_elems = s->max_rows * m->a.dim;
  s->p2p.timeout_ns = p2p_timeout_ns();
  // epochs start at 1 (the region is zero-initialised, so no word carries a live epoch)
  int rc = launch_kernel(Launcher{s->stream, LAUNCH_PLAIN, &s->launches}, set_p2p_epoch_kernel, dim3(1), dim3(1), 0, s->st, 1u);
  if (rc) return rc;
  CU(cudaStreamSynchronize(s->stream));
  if (s->graph) { cudaGraphExecDestroy(s->graph); s->graph = nullptr; }
  s->graph_tried = false;
  s->p2p_ready = true;
  return 0;
}

// the captured decode graph bakes in the active sequence's cache pointers and the layer count
static void drop_graph(lnb_session* s) {
  if (s->graph) {
    cudaSetDevice(s->m->device);
    cudaStreamSynchronize(s->stream);
    cudaGraphExecDestroy(s->graph);
    s->graph = nullptr;
  }
  s->graph_tried = false;
}
// Chunked prefill (SURVEY 8f-4), an EXTENSION: the reference builds its causal mask as [S,S] and adds it to [32,S,T]
// scores (llamatransformer.go:128-136,469-473), which only broadcasts for startPos 0 -- so it can only prefill a prompt
// in one call.  With this switch a Forward of S > 1 tokens at startPos > 0 is accepted and uses the mask a correct [S,T]
// broadcast would give: query row s (absolute position startPos + s) sees the keys t <= startPos + s.  Every other
// operation is unchanged, so a prompt prefilled in chunks leaves bit-identical caches and logits (LNB_ACC_STRICT).
extern "C" int lnb_session_set_chunked_prefill(lnb_session* s, int on) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  std::lock_guard<std::mutex> lk(s->mu);
  s->allow_chunked = on != 0;
  return 0;
}
extern "C" int lnb_session_set_layer_limit(lnb_session* s, int n) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  std::lock_guard<std::mutex> lk(s->mu);
  if (n != s->layer_limit) drop_graph(s);
  s->layer_limit = n;
  return 0;
}
extern "C" int64_t lnb_session_launch_count(lnb_session* s) { return s ? s->launches : 0; }
extern "C" int lnb_session_sync(lnb_session* s) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  CU(cudaSetDevice(s->m->device));
  CU(cudaStreamSynchronize(s->stream));
  return 0;
}

// peer all-reduce health: the flag travels with the call's own read-backs (enqueue before the stream sync, test after it)
static int p2p_err_enqueue(lnb_session* s) {
  if (s->p2p_ready) CU(cudaMemcpyAsync(s->h_err, &s->st->ar_error, 4, cudaMemcpyDeviceToHost, s->stream));
  return 0;
}
static int p2p_err_check(lnb_session* s) {
  if (!s->p2p_ready || *s->h_err == 0u) return 0;
  const uint32_t e = *s->h_err;
  return fail(LNB_ETIMEOUT, "peer all-reduce timed out after %llu ms: rank %d never received the words of rank %u for all-reduce #%u "
              "(a peer is late, dead or drives its session differently); the session's peer path is poisoned -- "
              "re-import the handles (lnb_session_p2p_import) or fall back with lnb_session_p2p_disable",
              (unsigned long long)(s->p2p.timeout_ns / 1000000ull), s->m->tp_rank, e & 15u, (e >> 4) & 0xffffffu);
}
extern "C" int lnb_session_p2p_disable(lnb_session* s) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(s->m->device));
  CU(cudaStreamSynchronize(s->stream));
  drop_graph(s);
  s->p2p_ready = false;   // the region stays mapped (peers may still write); every later call uses ncclAllReduce
  *s->h_err = 0;
  return 0;
}

static int ensure_logits(lnb_session* s, size_t rows) {
  if (s->logits_rows >= rows) return 0;
  cudaFree(s->logits);
  cudaFree(s->logits_full);
  s->logits = s->logits_full = nullptr;
  s->logits_rows = 0;
  CU(cudaMalloc((void**)&s->logits, rows * (size_t)s->m->vocab_l * 4));
  if (s->m->tp_size > 1) CU(cudaMalloc((void**)&s->logits_full, rows * (size_t)s->m->a.vocab_size * 4));
  s->logits_rows = rows;
  return 0;
}
// tensor-parallel: rows [row0, row0 + rows) of every rank's logits shard -> the same rows of logits_full (a collective)
static int gather_logits(lnb_session* s, int row0, int rows) {
  lnb_model* m = s->m;
  if (m->tp_size == 1) return 0;
  for (int r = row0; r < row0 + rows; r++)
    NC(g_nccl.AllGather(s->logits + (size_t)r * m->vocab_l, s->logits_full + (size_t)r * m->a.vocab_size, m->vocab_l, ncclFloat32_,
                        m->comm, s->stream));
  return 0;
}
// tensor-parallel LM head over NCCL: max-reduce the ranks' argmax keys, then publish the token (publish_kernel)
static int reduce_argmax_publish(const Launcher& L, lnb_session* s, bool advance) {
  NC(g_nccl.AllReduce(&s->st->amax_key, &s->st->amax_key, 1, ncclUint64_, ncclMax_, s->m->comm, s->stream));
  return launch_kernel(L, publish_kernel, dim3(1), dim3(1), 0, s->st, advance ? 1 : 0, s->d_tok_out);
}

// ---- persistent decode engine (engine.cuh) ---------------------------------------------------------------------
static float attn_scale_bf16(int head_dim) {  // dtype.BFloat16fromFloat32(float32(math.Sqrt(float64(HeadDim)))) :464
  float f = (float)sqrt((double)head_dim);
  uint32_t u;
  memcpy(&u, &f, 4);
  u &= 0xffff0000u;
  memcpy(&f, &u, 4);
  return f;
}
// Can this session's S=1 steps run as ONE persistent kernel?  (LNB_ENGINE=0 forces the kernel chain.)
static bool engine_probe(lnb_session* s) {
  if (s->eng_state) return s->eng_state > 0;
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  auto no = [&](const char* why) { s->eng_state = -1; s->eng_why = why; return false; };
  // Default: the engine is meant for where launch count or the serial order dominates -- LNB_ACC_STRICT at every N and
  // every host-driven loop; in LNB_ACC_FAST it competes with the kernel chain.  It is the default except for single-GPU
  // FAST sessions; LNB_ENGINE=1 / 0 forces it on / off.
  const char* e = getenv("LNB_ENGINE");
  if (e && !strcmp(e, "0")) return no("LNB_ENGINE=0");
  // single-sequence steps of single-GPU FAST sessions stay on the kernel chain by default (the batch engine does not care)
  s->eng_single_default = (e && !strcmp(e, "1")) || !(s->mode == LNB_ACC_FAST && m->tp_size == 1);
  const int kmax = std::max(a.dim, std::max(m->q_l, m->ffn_l));
  if ((size_t)kmax * 4 > (size_t)ENG_XMAX) return no("activation vector exceeds the engine's shared-memory work area");
  if (a.dim % 8 || m->q_l % 8 || m->ffn_l % 8) return no("widths must be multiples of 8");
  if ((size_t)a.dim * 8 > (size_t)ENG_XMAX) return no("dim too wide for the engine's RMSNorm prologue");
  const int n_rep = a.n_heads / a.n_kv_heads;
  if (a.head_dim > 128 || a.head_dim % 8 || n_rep > 8) return no("head shape");
  if (eng_sdpa_smem(s->seq_len, a.head_dim, n_rep) > (size_t)ENG_WORK) return no("SequenceLength too long for the in-engine attention phase");
  int ch, nt;
  if (s->mode == LNB_ACC_STRICT && !eng_scan_shape(a.dim, &ch, &nt)) return no("dim does not fit the engine's binade scan");
  if (m->q_l / a.head_dim > m->sm_count) return no("more query heads than SMs");
  int occ = 0;
  cudaError_t ce;
  if (s->mode == LNB_ACC_STRICT) {
    ce = cudaFuncSetAttribute(decode_engine_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENG_SMEM);
    if (ce == cudaSuccess) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, decode_engine_kernel<1>, ENG_THREADS, ENG_SMEM);
  } else {
    ce = cudaFuncSetAttribute(decode_engine_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENG_SMEM);
    if (ce == cudaSuccess) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, decode_engine_kernel<8>, ENG_THREADS, ENG_SMEM);
  }
  if (ce != cudaSuccess || occ < 1) { cudaGetLastError(); return no("the engine kernel does not fit an SM"); }
  if (cudaMalloc((void**)&s->d_bar, 256) != cudaSuccess) { cudaGetLastError(); return no("cudaMalloc"); }
  {
    cudaError_t e2 = cudaMalloc((void**)&s->x_t, (size_t)a.dim * 4);
    if (e2 == cudaSuccess) e2 = cudaMalloc((void**)&s->h1_t, (size_t)a.dim * 4);
    if (e2 == cudaSuccess) e2 = cudaMalloc((void**)&s->qkv_t, (size_t)(m->q_l + 2 * m->kv_l) * 4);
    if (e2 == cudaSuccess) e2 = cudaMalloc((void**)&s->o_t, (size_t)m->q_l * 4);
    if (e2 == cudaSuccess) e2 = cudaMalloc((void**)&s->m_t, (size_t)m->ffn_l * 4);
    if (e2 != cudaSuccess) { cudaGetLastError(); return no("cudaMalloc"); }
    s->eng_tag = 0;   // forces the zero-fill of the tagged vectors before the first launch
  }
  {
    const char* pe = getenv("LNB_ENGINE_PROF");
    if (pe && strcmp(pe, "0")) {
      const size_t nb = (size_t)m->sm_count * ENG_NPROF * 8;
      if (cudaMalloc((void**)&s->d_prof, nb) == cudaSuccess) cudaMemset(s->d_prof, 0, nb);
      else { s->d_prof = nullptr; cudaGetLastError(); }
    }
  }
  s->eng_state = 1;
  return true;
}
// the engine needs the peer all-reduce under tensor parallelism (NCCL calls cannot be issued from inside a kernel)
static bool engine_capable(lnb_session* s) { return engine_probe(s) && (s->m->tp_size == 1 || s->p2p_ready); }
static bool engine_ok(lnb_session* s) { return engine_capable(s) && s->eng_single_default; }

// LNB_ACC_FAST prompt attention on the tensor cores (sdpa_tc.cuh); LNB_SDPA_TC=0 keeps the FMA-pipe tile kernel
// exp of every bf16 value as f64, per device (sdpa_tc.cuh); NULL on failure
static const double* exp_table_device() {
  static std::mutex mu;
  static double* tab[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lk(mu);
  if (!tab[dev]) {
    double* t = nullptr;
    if (cudaMalloc((void**)&t, 65536 * sizeof(double)) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    exp_tab_kernel<<<256, 256>>>(t);
    if (cudaDeviceSynchronize() != cudaSuccess) { cudaGetLastError(); cudaFree(t); return nullptr; }
    tab[dev] = t;
  }
  return tab[dev];
}
static bool sdpa_tc_enabled() {
  const char* e = getenv("LNB_SDPA_TC");
  return !(e && !strcmp(e, "0"));
}
static int eng_kt(int mode, int N, int K, int G) {
  const int per = (N / 8 + G - 1) / G;                      // most panels one CTA owns
  const int PT = mode == LNB_ACC_STRICT ? EngCfg<1>::kPT : EngCfg<8>::kPT;
  const int maxp = std::max(1, std::min(PT, per));
  // the largest of 512 / 256 / 128 / 64 whose tile (maxp panels x kt x 16 B) fits a 32 KB stage: few, large bulk copies, and
  // k-tiles the STRICT chain can unroll completely (eng_chain_tile<NG>)
  int kt = 512;
  while (kt > 64 && maxp * kt * 16 > EngCfg<1>::kStage) kt >>= 1;
  return std::min(kt, K);
}
// The packed copies the STRICT decode engine streams for w1|w3 and the LM head (wpack.cuh, DESIGN §4): built once per
// model, on its device, from the panel-major bf16.  If the memory is not there the engine streams bf16 (same bits).
static bool ensure_wpack(lnb_model* m) {
  std::lock_guard<std::mutex> lk(m->wpack_mu);
  if (m->wpack_state) return m->wpack_state > 0;
  if (cudaSetDevice(m->device) != cudaSuccess) { cudaGetLastError(); return false; }
  const lnb_model_args& a = m->a;
  const int G = m->sm_count, L = a.n_layers;
  auto no = [&](const std::string& why) { m->wpack_state = -1; m->wpack_why = why; return false; };
  struct Mat { const uint16_t* W; int N; lnb_model::WPack* wp; };
  std::vector<Mat> mats;
  m->wp_w13.assign(L, lnb_model::WPack{});
  for (int l = 0; l < L; l++) mats.push_back({m->layers[l].w13, 2 * m->ffn_l, &m->wp_w13[l]});
  mats.push_back({m->output, m->vocab_l, &m->wp_out});
  const int K = a.dim;
  size_t total = 0;
  std::vector<size_t> off_data, off_units;
  for (Mat& x : mats) {
    const int kt = eng_kt(LNB_ACC_STRICT, x.N, K, G);
    if (K % 32 || kt % 32) return no("packed weights need K and the k-tile to be multiples of 32");
    x.wp->kt = kt;
    x.wp->n_units = (int64_t)(x.N / 8) * ((K + kt - 1) / kt);
    off_data.push_back(total);
    total += (size_t)x.N / 8 * K * 12;
    off_units.push_back(total);
    total = (total + x.wp->n_units + 255) & ~(size_t)255;
  }
  unsigned long long* ctr = nullptr;
  if (cudaMalloc(&m->wpack_mem, total) != cudaSuccess || cudaMalloc((void**)&ctr, mats.size() * 16) != cudaSuccess) {
    cudaGetLastError();
    cudaFree(m->wpack_mem);
    m->wpack_mem = nullptr;
    char why[160];
    snprintf(why, sizeof(why), "cudaMalloc of the %.2f GB packed weight copy failed: the engine streams bf16", total / 1e9);
    return no(why);
  }
  cudaMemset(ctr, 0, mats.size() * 16);
  for (size_t i = 0; i < mats.size(); i++) {
    lnb_model::WPack& wp = *mats[i].wp;
    wp.data = static_cast<uint8_t*>(m->wpack_mem) + off_data[i];
    wp.units = static_cast<uint8_t*>(m->wpack_mem) + off_units[i];
    wpack_encode_kernel<<<G * 8, 256>>>(mats[i].W, mats[i].N / 8, K, wp.kt, wp.data, wp.units, ctr + 2 * i);
  }
  std::vector<unsigned long long> h(mats.size() * 2);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(h.data(), ctr, h.size() * 8, cudaMemcpyDeviceToHost);
  cudaFree(ctr);
  if (e != cudaSuccess) {
    cudaFree(m->wpack_mem);
    m->wpack_mem = nullptr;
    return no(std::string("packing the weights failed: ") + cudaGetErrorString(e));
  }
  for (size_t i = 0; i < mats.size(); i++) {
    mats[i].wp->read_bytes = (int64_t)h[2 * i];
    mats[i].wp->packed_units = (int64_t)h[2 * i + 1];
  }
  m->wpack_state = 1;
  return true;
}
extern "C" int lnb_model_wpack_read(lnb_model* m, int layer, uint8_t* data, uint8_t* units, uint16_t* src, int64_t* info) {
  if (!m) return fail(LNB_EINVAL, "model is NULL");
  if (!m->finalized) return fail(LNB_ESTATE, "model is not finalized");
  if (layer < -1 || layer >= m->a.n_layers) return fail(LNB_EINVAL, "layer %d out of range", layer);
  CU(cudaSetDevice(m->device));
  if (!ensure_wpack(m)) { g_err = m->wpack_why; return 0; }
  const lnb_model::WPack& wp = layer < 0 ? m->wp_out : m->wp_w13[layer];
  const int64_t N = layer < 0 ? m->vocab_l : 2 * (int64_t)m->ffn_l, K = m->a.dim;
  if (data) CU(cudaMemcpy(data, wp.data, (size_t)(N / 8) * K * 12, cudaMemcpyDeviceToHost));
  if (units) CU(cudaMemcpy(units, wp.units, (size_t)wp.n_units, cudaMemcpyDeviceToHost));
  if (src) CU(cudaMemcpy(src, layer < 0 ? m->output : m->layers[layer].w13, (size_t)N * K * 2, cudaMemcpyDeviceToHost));
  if (info) { info[0] = wp.kt; info[1] = wp.n_units; info[2] = wp.packed_units; info[3] = wp.read_bytes; info[4] = N; }
  return 1;
}
// kind -1: the full step; 0..4: independent copies of one projection of every layer (kernel-alone timing, plain buffers)
static int engine_build(lnb_session* s, int kind, const float* logits_out) {
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  const int n_layers = active_layers(s);
  if (s->d_phases && s->eng_key_seq == s->active_seq && s->eng_key_layers == n_layers && s->eng_key_kind == kind &&
      s->eng_key_logits == logits_out)
    return 0;
  const int G = m->sm_count, mode = s->mode;
  const size_t cache_off = (size_t)s->active_seq * s->seq_len * m->kv_l;
  const bool full = kind < 0;
  std::vector<EnginePhase> ph;
  // which phase of the step wrote a tagged vector last (consumers wait for exactly that phase's tag)
  int w_x = -1, w_h1 = -1, w_qkv = -1, w_o = -1, w_m = -1;
  auto gemv = [&](int pro, int epi, const uint16_t* W, int N, int K, const uint16_t* x, const uint16_t* norm_w, uint16_t* out, int ldo,
                  const uint16_t* res) {
    EnginePhase e{};
    e.type = EP_GEMV; e.pro = pro; e.epi = epi; e.W = W; e.N = N; e.K = K; e.kt = eng_kt(mode, N, K, G); e.x = x; e.ldx = K;
    e.norm_w = norm_w; e.out_bf16 = out; e.ldo = ldo; e.res = res;
    return e;
  };
  auto input = [&](EnginePhase& e, const uint32_t* vec, int writer) {   // tagged input of the phase being appended
    if (full && writer >= 0) { e.x_t = vec; e.x_delta = (int)ph.size() - writer; }
  };
  auto resid = [&](EnginePhase& e, const uint32_t* vec, int writer) {
    if (full && writer >= 0) { e.res_t = vec; e.res_delta = (int)ph.size() - writer; }
  };
  const bool tp = m->tp_size > 1;
  // STRICT streams the packed copies of w1|w3 and the LM head (the FAST engine's KS = 8 chains read bf16 only)
  const bool wpack = mode == LNB_ACC_STRICT && ensure_wpack(m);
  auto packed = [&](EnginePhase& e, const lnb_model::WPack& wp) {
    if (wpack && wp.kt == e.kt) { e.Wp = wp.data; e.Wu = wp.units; }
  };
  for (int l = 0; l < n_layers; l++) {
    LayerW& W = m->layers[l];
    if (full || kind == 0) {  // attn_norm -> wq|wk|wv -> RoPE -> KV append
      EnginePhase e = gemv(PRO_RMSNORM, EPI_QKV_ROPE, W.wqkv, m->q_l + 2 * m->kv_l, a.dim, s->x, W.attn_norm, s->q, m->q_l, nullptr);
      e.q_dim = m->q_l; e.kv_dim = m->kv_l; e.cache_k = s->ck[l] + cache_off; e.cache_v = s->cv[l] + cache_off;
      if (full && l == 0) e.flags |= EF_X_TOKEN;
      else input(e, s->x_t, w_x);
      if (full) { e.out_t = s->qkv_t; w_qkv = (int)ph.size(); }
      ph.push_back(e);
    }
    if (full) {
      EnginePhase e{};
      e.type = EP_SDPA; e.kv_dim = m->kv_l; e.q_dim = m->q_l;
      e.cache_k = s->ck[l] + cache_off; e.cache_v = s->cv[l] + cache_off;
      input(e, s->qkv_t, w_qkv);
      e.out_t = s->o_t; w_o = (int)ph.size();
      ph.push_back(e);
    }
    if (full || kind == 1) {  // wo + residual
      EnginePhase e = gemv(PRO_PLAIN, (tp && full) ? EPI_P2P : EPI_RESID, W.wo, a.dim, m->q_l, s->o, nullptr, s->h1, a.dim, s->x);
      input(e, s->o_t, w_o);
      if (full && !tp) {
        if (l == 0) e.flags |= EF_RES_TOKEN; else resid(e, s->x_t, w_x);
        e.out_t = s->h1_t; w_h1 = (int)ph.size();
      }
      ph.push_back(e);
      if (tp && full) {
        EnginePhase r{};
        r.type = EP_REDUCE;
        if (l == 0) r.flags |= EF_RES_TOKEN; else resid(r, s->x_t, w_x);
        r.out_t = s->h1_t; w_h1 = (int)ph.size();
        ph.push_back(r);
      }
    }
    if (full || kind == 2) {  // ffn_norm -> w1|w3 -> SiLU * up
      EnginePhase e = gemv(PRO_RMSNORM, EPI_SWIGLU, W.w13, 2 * m->ffn_l, a.dim, s->h1, W.ffn_norm, s->mbuf, m->ffn_l, nullptr);
      packed(e, m->wp_w13[l]);
      input(e, s->h1_t, w_h1);
      if (full) { e.out_t = s->m_t; w_m = (int)ph.size(); }
      ph.push_back(e);
    }
    if (full || kind == 3) {  // w2 + residual
      EnginePhase e = gemv(PRO_PLAIN, (tp && full) ? EPI_P2P : EPI_RESID, W.w2, a.dim, m->ffn_l, s->mbuf, nullptr, s->x, a.dim, s->h1);
      input(e, s->m_t, w_m);
      if (full && !tp) { resid(e, s->h1_t, w_h1); e.out_t = s->x_t; w_x = (int)ph.size(); }
      ph.push_back(e);
      if (tp && full) {
        EnginePhase r{};
        r.type = EP_REDUCE;
        resid(r, s->h1_t, w_h1);
        r.out_t = s->x_t; w_x = (int)ph.size();
        ph.push_back(r);
      }
    }
  }
  if (full || kind == 4) {
    const int reps = kind == 4 ? 4 : 1;
    for (int i = 0; i < reps; i++) {
      EnginePhase e = gemv(PRO_RMSNORM, EPI_LOGITS, m->output, m->vocab_l, a.dim, s->x, m->norm, nullptr, m->vocab_l, nullptr);
      packed(e, m->wp_out);
      e.out_f32 = const_cast<float*>(logits_out); e.n_offset = m->tp_rank * m->vocab_l;
      if (full && n_layers > 0) input(e, s->x_t, w_x);
      if (full) e.flags |= EF_GRID_SYNC;
      ph.push_back(e);
    }
    if (full && tp) {
      EnginePhase r{};
      r.type = EP_ARGMAX;
      ph.push_back(r);
    }
  }
  if (!full) ph.back().flags |= EF_GRID_SYNC;   // one barrier per sweep keeps the CTAs of a timing run together
  if ((int)ph.size() > s->phases_cap) {
    cudaFree(s->d_phases);
    s->d_phases = nullptr;
    s->phases_cap = 0;
    CU(cudaMalloc((void**)&s->d_phases, ph.size() * sizeof(EnginePhase)));
    s->phases_cap = (int)ph.size();
  }
  CU(cudaStreamSynchronize(s->stream));   // a running engine may still read the old list
  CU(cudaMemcpy(s->d_phases, ph.data(), ph.size() * sizeof(EnginePhase), cudaMemcpyHostToDevice));
  s->n_phases = (int)ph.size();
  s->eng_key_seq = s->active_seq; s->eng_key_layers = n_layers; s->eng_key_kind = kind; s->eng_key_logits = logits_out;
  return 0;
}
// n_steps S=1 forwards; the first input token and position come from the device state (set_state_kernel).  One launch
// covers up to 65535 / n_phases steps (16-bit activation tags); longer runs continue from the device state.
static int engine_launch(lnb_session* s, int n_steps, bool advance) {
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  EngineParams P{};
  P.phases = s->d_phases; P.n_phases = s->n_phases; P.st = s->st;
  P.emb = m->tok_embd; P.dim = a.dim; P.head_dim = a.head_dim; P.n_rep = a.n_heads / a.n_kv_heads; P.seq_len = s->seq_len;
  P.cis = m->cis; P.silu_tab = m->silu_tab; P.eps = a.norm_eps; P.attn_scale = attn_scale_bf16(a.head_dim);
  P.strict = s->mode == LNB_ACC_STRICT ? 1 : 0;
  P.tok_out = s->d_tok_out; P.bar_ctr = s->d_bar;
  P.p2p = s->p2p; P.tp = m->tp_size;
  P.timeout_ns = p2p_timeout_ns();
  P.err_host = s->h_err;
  {
    // L2 prefetch per CTA and projection beyond the ring: 132 x 256 KB = 33 MB of the 50 MB L2 when enabled (LNB_ENGINE_PF_KB, 0 = off)
    static const int pf_kb = [] { const char* e = getenv("LNB_ENGINE_PF_KB"); return e ? atoi(e) : 0; }();
    P.pf_window = pf_kb > 0 ? (unsigned int)pf_kb * 1024u : 0u;
  }
  P.prof = s->d_prof;
  P.advance = advance ? 1 : 0;
  const int max_steps = std::max(1, 65000 / std::max(1, s->n_phases));
  if (!advance && n_steps > max_steps) return fail(LNB_EINVAL, "engine: too many steps for one launch");
  for (int done = 0; done < n_steps;) {
    const int n = std::min(n_steps - done, max_steps);
    if (s->eng_tag == 0 || (uint64_t)s->eng_tag + (uint64_t)n * s->n_phases > 65535u) {
      // the 16-bit tags wrap: kill every old tag first (0 is never issued)
      CU(cudaMemsetAsync(s->x_t, 0, (size_t)a.dim * 4, s->stream));
      CU(cudaMemsetAsync(s->h1_t, 0, (size_t)a.dim * 4, s->stream));
      CU(cudaMemsetAsync(s->qkv_t, 0, (size_t)(m->q_l + 2 * m->kv_l) * 4, s->stream));
      CU(cudaMemsetAsync(s->o_t, 0, (size_t)m->q_l * 4, s->stream));
      CU(cudaMemsetAsync(s->m_t, 0, (size_t)m->ffn_l * 4, s->stream));
      s->eng_tag = 1;
    }
    P.n_steps = n;
    P.tag_base = s->eng_tag;
    s->eng_tag += (uint32_t)n * (uint32_t)s->n_phases;
    CU(cudaMemsetAsync(s->d_bar, 0, 4, s->stream));
    const int rc = launch_kernel(Launcher{s->stream, LAUNCH_COOP, &s->launches},
                                 s->mode == LNB_ACC_STRICT ? decode_engine_kernel<1> : decode_engine_kernel<8>, dim3(m->sm_count),
                                 dim3(ENG_THREADS), ENG_SMEM, P);
    if (rc) return rc;
    done += n;
  }
  s->last_was_engine = true;
  return 0;
}
// after a failed stream sync: did the engine trap, and why?
static int engine_fault(lnb_session* s, cudaError_t e) {
  const uint32_t c = s->h_err ? *s->h_err : 0u;
  if ((c >> 28) == 0x8u)
    return fail(LNB_ETIMEOUT, "peer all-reduce timed out inside the decode engine: rank %d never received the words of rank %u for "
                "all-reduce #%u (a peer is late or dead); the kernel trapped, this process's CUDA context is gone (%s)",
                s->m->tp_rank, c & 15u, (c >> 4) & 0xffffffu, cudaGetErrorString(e));
  if ((c >> 28) == 0xCu) return fail(LNB_ECUDA, "decode engine: a CTA never reached grid barrier target %u (%s)", c & 0xffffffu, cudaGetErrorString(e));
  if ((c >> 28) == 0xDu) return fail(LNB_ECUDA, "decode engine: weight stage %u never completed (%s)", c & 0xffffffu, cudaGetErrorString(e));
  if ((c >> 28) == 0xEu) return fail(LNB_ECUDA, "decode engine: the activations tagged %u never arrived (%s)", c & 0xffffu, cudaGetErrorString(e));
  return fail(LNB_ECUDA, "stream synchronize failed: %s", cudaGetErrorString(e));
}

// ---- batch engine (engine_batch.cuh): one launch advances all sequences of a batched session by one token -------------------
static bool batch_engine_usable(lnb_session* s) {
  if (!engine_capable(s)) return false;
  const lnb_model_args& a = s->m->a;
  if ((size_t)a.dim * 4 > 16 * 1024) return false;                      // norm weights as f32 in 16 KB of shared memory
  const char* e = getenv("LNB_BATCH_ENGINE");
  if (e && !strcmp(e, "0")) return false;
  return true;
}
static bool batch_engine_ok(lnb_session* s) { return s->n_seq >= 2 && batch_engine_usable(s); }
// speculative verification: a call of >= 2 rows runs the batch engine, single-sequence sessions included (engine_capable
// already holds every position below the engine's limit, eng_sdpa_smem)
static bool spec_engine_ok(lnb_session* s, int rows) { return rows >= 2 && batch_engine_usable(s); }
static int batch_engine_build(lnb_session* s, const float* logits_out) {
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  const int n_layers = active_layers(s);
  if (s->d_bphases && s->bkey_layers == n_layers && s->bkey_logits == logits_out) return 0;
  if (!s->bx) {
    cudaError_t e = cudaMalloc((void**)&s->bx, (size_t)a.dim * 16);
    if (e == cudaSuccess) e = cudaMalloc((void**)&s->bh1, (size_t)a.dim * 16);
    if (e == cudaSuccess) e = cudaMalloc((void**)&s->bq, (size_t)m->q_l * 16);
    if (e == cudaSuccess) e = cudaMalloc((void**)&s->bo, (size_t)m->q_l * 16);
    if (e == cudaSuccess) e = cudaMalloc((void**)&s->bm, (size_t)m->ffn_l * 16);
    if (e == cudaSuccess) e = cudaMalloc((void**)&s->d_bkeys, 64);
    if (e == cudaSuccess) e = cudaMalloc((void**)&s->bxn, (size_t)a.dim * 16);
    if (e != cudaSuccess) return fail(LNB_ENOMEM, "batch engine buffers: %s", cudaGetErrorString(e));
    CU(cudaMemset(s->bx, 0, (size_t)a.dim * 16)); CU(cudaMemset(s->bh1, 0, (size_t)a.dim * 16));
    CU(cudaMemset(s->bq, 0, (size_t)m->q_l * 16)); CU(cudaMemset(s->bo, 0, (size_t)m->q_l * 16));
    CU(cudaMemset(s->bm, 0, (size_t)m->ffn_l * 16)); CU(cudaMemset(s->bxn, 0, (size_t)a.dim * 16));
    // FAST: the FMA-pipe kernel by default -- on an H100 (3.35 TB/s) it keeps up with the weight stream at 8 rows and beat
    // the tensor-core form, 880 vs 602 tokens/s (bench.py --config batch8 --acc fast, H100 SXM 700 W); LNB_BATCH_TC=1 selects
    // the tensor-core form (every K a multiple of 16)
    {
      const char* e2 = getenv("LNB_BATCH_TC");
      s->batch_tc = s->mode != LNB_ACC_STRICT && (e2 && !strcmp(e2, "1")) && a.dim % 16 == 0 && m->q_l % 16 == 0 && m->ffn_l % 16 == 0;
    }
    if (s->mode == LNB_ACC_STRICT) CU(cudaFuncSetAttribute(batch_engine_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENG_SMEM));
    else if (s->batch_tc) CU(cudaFuncSetAttribute(batch_engine_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, BT_SMEM));
    else CU(cudaFuncSetAttribute(batch_engine_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, ENG_SMEM));
  }
  const int G = m->sm_count, mode = s->mode;
  const bool tp = m->tp_size > 1;
  const bool tc = s->batch_tc != 0;
  std::vector<BatchPhase> ph;
  auto gemv = [&](int pro, int epi, const uint16_t* W, int N, int K, const uint16_t* x, const uint16_t* norm_w, uint16_t* out, int ldo,
                  const uint16_t* res) {
    BatchPhase e{};
    e.type = BP_GEMV; e.pro = pro; e.epi = epi; e.W = W; e.N = N; e.K = K; e.kt = eng_kt(mode, N, K, G); e.x = x;
    e.norm_w = norm_w; e.out = out; e.ldo = ldo; e.res = res;
    if (tc) {
      // tensor-core form: 128-row tiles; the k-tile grows as the CTA's share of the rows shrinks (about 32 KB per stage,
      // copies of 2 .. 8 KB); RMSNorm happened in the SCALE phase (x = the normalised row)
      const int per = std::max(1, std::min(16, (N / 8 + G - 1) / G));
      int kt = BT_KT_MAX;
      while (kt > 128 && per * kt * 16 > EngCfg<1>::kStage) kt >>= 1;
      e.kt = std::min(kt, K);
      if (pro == PRO_RMSNORM) { e.pro = PRO_PLAIN; e.x = s->bxn; e.norm_w = nullptr; }
    }
    return e;
  };
  auto scale = [&](const uint16_t* x, bool from_token, const uint16_t* norm_w) {
    BatchPhase e{};
    e.type = BP_SCALE; e.K = a.dim; e.x = x; e.out = s->bx; e.flags = from_token ? EF_X_TOKEN : 0;
    if (tc) { e.norm_w = norm_w; e.xn = s->bxn; }
    return e;
  };
  auto reduce = [&](const uint16_t* res, uint16_t* out) {
    BatchPhase e{};
    e.type = BP_REDUCE; e.res = res; e.out = out;
    return e;
  };
  for (int l = 0; l < n_layers; l++) {
    LayerW& W = m->layers[l];
    ph.push_back(scale(s->bx, l == 0, W.attn_norm));
    {
      BatchPhase e = gemv(PRO_RMSNORM, EPI_QKV_ROPE, W.wqkv, m->q_l + 2 * m->kv_l, a.dim, s->bx, W.attn_norm, s->bq, m->q_l, nullptr);
      e.q_dim = m->q_l; e.kv_dim = m->kv_l; e.cache_k = s->ck[l]; e.cache_v = s->cv[l];
      ph.push_back(e);
    }
    {
      BatchPhase e{};
      e.type = BP_SDPA; e.x = s->bq; e.out = s->bo; e.q_dim = m->q_l; e.kv_dim = m->kv_l; e.cache_k = s->ck[l]; e.cache_v = s->cv[l];
      ph.push_back(e);
    }
    ph.push_back(gemv(PRO_PLAIN, tp ? EPI_P2P : EPI_RESID, W.wo, a.dim, m->q_l, s->bo, nullptr, s->bh1, a.dim, s->bx));
    if (tp) ph.push_back(reduce(s->bx, s->bh1));
    ph.push_back(scale(s->bh1, false, W.ffn_norm));
    ph.push_back(gemv(PRO_RMSNORM, EPI_SWIGLU, W.w13, 2 * m->ffn_l, a.dim, s->bh1, W.ffn_norm, s->bm, m->ffn_l, nullptr));
    ph.push_back(gemv(PRO_PLAIN, tp ? EPI_P2P : EPI_RESID, W.w2, a.dim, m->ffn_l, s->bm, nullptr, s->bx, a.dim, s->bh1));
    if (tp) ph.push_back(reduce(s->bh1, s->bx));
  }
  ph.push_back(scale(s->bx, n_layers == 0, m->norm));
  {
    BatchPhase e = gemv(PRO_RMSNORM, EPI_LOGITS, m->output, m->vocab_l, a.dim, s->bx, m->norm, nullptr, m->vocab_l, nullptr);
    e.out_f32 = const_cast<float*>(logits_out); e.n_offset = m->tp_rank * m->vocab_l;
    ph.push_back(e);
  }
  {
    BatchPhase e{};
    e.type = BP_TOKENS;
    ph.push_back(e);
  }
  cudaFree(s->d_bphases);
  s->d_bphases = nullptr;
  CU(cudaMalloc((void**)&s->d_bphases, ph.size() * sizeof(BatchPhase)));
  CU(cudaStreamSynchronize(s->stream));
  CU(cudaMemcpy(s->d_bphases, ph.data(), ph.size() * sizeof(BatchPhase), cudaMemcpyHostToDevice));
  s->n_bphases = (int)ph.size();
  s->bkey_layers = n_layers; s->bkey_logits = logits_out;
  return 0;
}
// n rows: token tokens[m] at position pos_arr[m] on the cache of sequence row_seq[m] (NULL: sequence m), already on the device
static int batch_engine_launch(lnb_session* s, int n, const int32_t* tokens, const int32_t* pos_arr, const int32_t* row_seq) {
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  BatchParams P{};
  P.phases = s->d_bphases; P.n_phases = s->n_bphases; P.n = n; P.st = s->st;
  P.emb = m->tok_embd; P.dim = a.dim; P.head_dim = a.head_dim; P.n_rep = a.n_heads / a.n_kv_heads; P.seq_len = s->seq_len;
  P.cis = m->cis; P.silu_tab = m->silu_tab; P.eps = a.norm_eps; P.attn_scale = attn_scale_bf16(a.head_dim);
  P.strict = s->mode == LNB_ACC_STRICT ? 1 : 0;
  P.tokens = tokens; P.pos_arr = pos_arr; P.row_seq = row_seq; P.cache_seq_stride = (long long)s->seq_len * m->kv_l;
  P.rscale = s->rs; P.keys = s->d_bkeys; P.next_arr = s->d_next_arr; P.bar_ctr = s->d_bar;
  P.p2p = s->p2p; P.tp = m->tp_size;
  P.timeout_ns = p2p_timeout_ns();
  P.err_host = s->h_err;
  P.prof = s->d_prof;
  *s->h_err = 0;
  CU(cudaMemsetAsync(s->d_bar, 0, 4, s->stream));
  CU(cudaMemsetAsync(s->d_bkeys, 0, 64, s->stream));
  const auto kern = s->mode == LNB_ACC_STRICT ? batch_engine_kernel<1> : s->batch_tc ? batch_engine_kernel<0> : batch_engine_kernel<8>;
  const int rc = launch_kernel(Launcher{s->stream, LAUNCH_COOP, &s->launches}, kern, dim3(m->sm_count), dim3(ENG_THREADS),
                               s->batch_tc ? BT_SMEM : ENG_SMEM, P);
  if (rc) return rc;
  s->last_was_engine = false;
  return 0;
}

static int sync_stream(lnb_session* s) {
  cudaError_t e = cudaStreamSynchronize(s->stream);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return engine_fault(s, e);
  return 0;
}
// one S=1 forward through the engine; the token travels in the device state (set_state_kernel)
static int enqueue_decode_engine(lnb_session* s, int32_t token, int start_pos, int n_steps, bool advance, bool reset_step, const float* logits_out) {
  int rc = engine_build(s, -1, logits_out);
  if (rc) return rc;
  if ((rc = set_state(s, start_pos, 1, token, reset_step))) return rc;
  *s->h_err = 0;
  return engine_launch(s, n_steps, advance);
}

// The rows of one forward: where row r's token, position and KV cache come from, and what the LM head makes of them.
// rows_single, rows_batch, rows_ragged and rows_spec are the only places that decide this; the forward builders read it from
// here.
enum RowsKind { ROWS_SINGLE, ROWS_BATCH, ROWS_RAGGED, ROWS_SPEC };
// what the LM head produces: the last row's greedy token with no logits kept, the last row's or every row's (NONE, LAST,
// ALL); or, for output rows that each end their own sequence, the logits and a greedy token in d_next_arr per row (PER_ROW)
enum RowsHead { HEAD_NONE, HEAD_LAST, HEAD_ALL, HEAD_PER_ROW };
struct Rows {
  RowsKind kind;
  int S;
  const int32_t* tokens;    // device token id of each row, or NULL: st->next_token (a device-driven decode step)
  const int32_t* pos_arr;   // device position of each row, or NULL: st->pos + r
  const int32_t* row_seq;   // ragged, speculative: the sequence of each row
  size_t cache_off;         // elements to the cache every row addresses (the active sequence's), or 0
  long long seq_stride;     // rows on several caches: elements between consecutive sequences' caches, else 0
  int mb_rows;              // launch_gemv's mb_rows: ragged 8, else 0
  const int32_t* seg_last;  // ragged: the last row of each segment
  RowsHead head;
  int head_rows;            // rows the LM head computes
  bool advance;             // the LM head advances st->pos and appends the token to d_tok_out (device-driven decode)
  bool gather;              // tensor-parallel: the kept logits are all-gathered for the host
  bool record;              // a row's sequence is penalized: the forward records every row's token in d_hist
};
// rows 0..S-1 of the active sequence at st->pos + r.  tokens: device ids, or NULL for st->next_token.  logits_rows: logits
// kept, 0 = none, 1 = the last row, S = all rows.
static Rows rows_single(const lnb_session* s, int S, const int32_t* tokens, int logits_rows, bool advance, bool gather) {
  Rows R{};
  R.kind = ROWS_SINGLE; R.S = S; R.tokens = tokens;
  R.cache_off = (size_t)s->active_seq * s->seq_len * s->m->kv_l;
  R.head = logits_rows == 0 ? HEAD_NONE : logits_rows == 1 ? HEAD_LAST : HEAD_ALL;
  R.head_rows = logits_rows > 1 ? S : 1;
  R.advance = advance; R.gather = gather;
  R.record = s->pen_on[s->active_seq];
  return R;
}
// a batched step: row r is sequence r, token d_tokens[r] at position d_pos_arr[r]
static Rows rows_batch(const lnb_session* s, int n) {
  Rows R{};
  R.kind = ROWS_BATCH; R.S = n; R.tokens = s->d_tokens; R.pos_arr = s->d_pos_arr;
  R.seq_stride = (long long)s->seq_len * s->m->kv_l;
  R.head = HEAD_PER_ROW; R.head_rows = n;
  for (int i = 0; i < n; i++) R.record |= s->pen_on[i];
  return R;
}
// a ragged call: the row map in d_rag, [tokens | row_seq | row_pos] of `rows` words each, then the last row of each segment
static Rows rows_ragged(const lnb_session* s, int rows, int n_segs, bool record) {
  Rows R{};
  R.kind = ROWS_RAGGED; R.S = rows; R.tokens = s->d_rag; R.row_seq = s->d_rag + rows; R.pos_arr = s->d_rag + 2 * rows;
  R.seq_stride = (long long)s->seq_len * s->m->kv_l;
  R.mb_rows = 8;
  R.seg_last = s->d_rag + 3 * rows;
  R.head = HEAD_PER_ROW; R.head_rows = n_segs;
  R.record = record;
  return R;
}
// a speculative verification call: the row map in d_rag, [tokens | row_seq | row_pos] of `rows` words each; consecutive
// rows of a segment are consecutive positions of one sequence, and EVERY row is an output row (its next token is compared
// with the following draft), so the LM head runs over all of them
static Rows rows_spec(const lnb_session* s, int rows, bool record) {
  Rows R{};
  R.kind = ROWS_SPEC; R.S = rows; R.tokens = s->d_rag; R.row_seq = s->d_rag + rows; R.pos_arr = s->d_rag + 2 * rows;
  R.seq_stride = (long long)s->seq_len * s->m->kv_l;
  R.head = HEAD_PER_ROW; R.head_rows = rows;
  R.record = record;
  return R;
}

// Attention of layer l for the rows R (queries in s->q), written to out: plain rows, or the X8 operand of the tensor-core
// Wo GEMM (out_x8).  Ragged rows always stream, so a ragged call has one attention path whatever the session's other calls
// use.  sdpa_tc_kernel and sdpa_prefill_kernel write X8 only; sdpa_decode_kernel writes plain rows only.
static int launch_attention(const Launcher& L, lnb_session* s, int l, const Rows& R, uint16_t* out, int out_x8) {
  const lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  const int S = R.S, n_rep = a.n_heads / a.n_kv_heads, n_q = m->q_l / a.head_dim, n_kv = m->kv_l / a.head_dim;
  const uint16_t *ck = s->ck[l] + R.cache_off, *cv = s->cv[l] + R.cache_off;
  const int32_t* pos_ptr = &s->st->pos;
  const float scale = attn_scale_bf16(a.head_dim);
  const int strict = s->mode == LNB_ACC_STRICT ? 1 : 0;
  // rows on a row -> position map (a batched step, or a speculative call whose rows follow each other in one sequence's
  // cache): the decode kernel within its fit, else the streamed kernels -- the attention a batched step of those rows runs
  const bool batched = R.kind == ROWS_BATCH || R.kind == ROWS_SPEC;
  auto streamed = [&]() {
    StreamAttn P{};
    P.q = s->q; P.ldq = m->q_l;
    P.cache_k = ck; P.cache_v = cv; P.kv_dim = m->kv_l;
    P.row_cache_stride = R.seq_stride; P.row_seq = R.row_seq; P.pos_arr = R.pos_arr;
    P.n_rep = n_rep; P.hd = a.head_dim; P.n_heads = n_q;
    P.pos_ptr = pos_ptr; P.pos_step = 1;
    P.out = out; P.ldo = m->q_l; P.out_x8 = out_x8;
    P.scale = scale; P.strict = strict;
    return launch_stream_attn(L, P, S, n_kv, s->ss);
  };
  if (R.kind == ROWS_RAGGED) return streamed();
  if (!out_x8 && (S == 1 || batched) && s->sdpa_smem_decode)
    return launch_kernel(L, sdpa_decode_kernel, dim3(n_kv, S), dim3(128 * n_rep), s->sdpa_decode_smem, (const uint16_t*)s->q, ck, cv,
                         m->kv_l, n_rep, a.head_dim, out, pos_ptr, s->seq_len, strict, scale, R.pos_arr,
                         (long long)s->seq_len * m->kv_l, m->q_l, (const LnbDevState*)s->st, R.row_seq);
  if (out_x8 && a.head_dim == SP_HD) {
    const double* exp_tab = sdpa_tc_enabled() ? exp_table_device() : nullptr;
    if (exp_tab)
      return launch_kernel(L, sdpa_tc_kernel, dim3(n_q, (S + 127) / 128), dim3(256), (size_t)ST_SMEM, (const uint16_t*)s->q, m->q_l, ck,
                           cv, m->kv_l, n_rep, out, m->q_l, pos_ptr, S, scale, exp_tab);
    return launch_kernel(L, sdpa_prefill_kernel, dim3(n_q, (S + SP_QB - 1) / SP_QB), dim3(256), (size_t)SP_SMEM, (const uint16_t*)s->q,
                         m->q_l, ck, cv, m->kv_l, n_rep, out, m->q_l, pos_ptr, S, scale);
  }
  if (batched || s->stream_attn) return streamed();
  return launch_kernel(L, sdpa_kernel, dim3(n_q, S), dim3(128), (size_t)s->seq_len * 12 + (size_t)a.head_dim * 4, (const uint16_t*)s->q,
                       m->q_l, ck, cv, m->kv_l, n_rep, a.head_dim, out, m->q_l, pos_ptr, 0, S, S > 1 ? 1 : 0, strict, scale, out_x8);
}

// LM head of a batched step or a ragged call, where every output row is the last row of its own sequence: ragged calls
// first compact the last row of each segment into h1 (dead after the last layer); then ONE EPI_LOGITS GEMV over the
// head_rows rows and one greedy argmax per row into d_next_arr (tensor-parallel: on the gathered logits)
static int per_row_head(const Launcher& L, lnb_session* s, const Rows& R) {
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  const bool strict = (s->mode == LNB_ACC_STRICT);
  const int n = R.head_rows;
  const uint16_t* x = R.seg_last ? s->h1 : s->x;
  int rc;
  if (R.seg_last && (rc = launch_kernel(L, gather_rows_kernel, dim3(n), dim3(256), 0, (const uint16_t*)s->x, R.seg_last,
                                        (const LnbDevState*)s->st, s->h1, a.dim)))
    return rc;
  if (strict && (rc = launch_rms_scale(L, x, a.dim, s->rs, n, a.dim, a.norm_eps))) return rc;
  GemvParams p{};
  p.rscale = strict ? s->rs : nullptr;
  p.W = m->output; p.N = m->vocab_l; p.K = a.dim; p.x = x; p.ldx = a.dim; p.norm_w = m->norm; p.eps = a.norm_eps;
  p.out_f32 = s->logits; p.ldo = m->vocab_l; p.n_offset = m->tp_rank * m->vocab_l; p.st = nullptr; p.argmax_row = -1;
  if ((rc = launch_gemv<PRO_RMSNORM, EPI_LOGITS>(L, s->mode, p, n, R.mb_rows))) return rc;
  if ((rc = gather_logits(s, 0, n))) return rc;
  const float* lg = (m->tp_size > 1) ? s->logits_full : s->logits;
  return launch_kernel(L, argmax_f32_kernel, dim3(n), dim3(256), 0, lg, a.vocab_size, s->d_next_arr);
}

// Prompt processing on the tensor cores (LNB_ACC_FAST, S >= 32): the same forward pass as
// enqueue_forward with every projection as a tensor-core GEMM (gemm_tc.cuh) and the elementwise steps
// as separate memory-bound kernels that write the next GEMM's X8 operand directly.  Batched steps (at most 8 rows)
// never qualify.
static bool forward_tc_ok(const lnb_session* s, int S) {
  const lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  return s->mode == LNB_ACC_FAST && s->xn8 && S >= 32 && (m->q_l + 2 * m->kv_l) % TC_BN == 0 && a.dim % TC_BN == 0 &&
         (2 * m->ffn_l) % TC_BN == 0 && a.dim % TC_KT == 0 && m->q_l % TC_KT == 0 && m->ffn_l % TC_KT == 0;
}
static int enqueue_forward_tc(lnb_session* s, const Rows& R);

// The history write of a forward over the rows R (R.record: a row's sequence is penalized), before anything advances
// st->pos.  token / pos0 (>= 0): the one row's token and position when they ride in a launch argument (the decode engine).
static int launch_record(lnb_session* s, const Rows& R, int32_t token = -1, int pos0 = -1) {
  if (!R.record) return 0;
  return launch_kernel(Launcher{s->stream, LAUNCH_PDL, &s->launches}, penalty_record_kernel, dim3((R.S + 255) / 256), dim3(256), 0,
                       s->d_hist, s->seq_len, (const LnbDevState*)s->st, R.tokens, R.pos_arr, R.row_seq,
                       R.kind == ROWS_SINGLE ? s->active_seq : -1, token, pos0, R.S);
}

// Enqueue one LlamaTransformer.Forward (llamatransformer.go:145-180) for the rows R on the session stream: on the tensor
// cores when forward_tc_ok, else as the kernel chain below.  Every forward but the decode engines' comes through here.
static int enqueue_forward(lnb_session* s, const Rows& R) {
  s->last_was_engine = false;   // this forward's residual stream is s->x
  if (const int rc = launch_record(s, R)) return rc;
  if (forward_tc_ok(s, R.S)) return enqueue_forward_tc(s, R);
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  const Launcher L{s->stream, LAUNCH_PDL, &s->launches};
  const int mode = s->mode;
  const int S = R.S, mb_rows = R.mb_rows;
  int rc;
  rc = launch_kernel(L, gather_rows_kernel, dim3(S), dim3(256), 0, (const uint16_t*)m->tok_embd, R.tokens, (const LnbDevState*)s->st, s->x,
                     a.dim);
  if (rc) return rc;
  const int n_layers = active_layers(s);
  const bool strict = (mode == LNB_ACC_STRICT);
  auto strict_scale = [&](const uint16_t* xin, int rows) -> int {
    if (!strict) return 0;
    return launch_rms_scale(L, xin, a.dim, s->rs, rows, a.dim, a.norm_eps);
  };
  // wo / w2 + residual: out = res + x W^T; tensor-parallel ranks sum their partials first (peer all-reduce or NCCL)
  auto proj_resid = [&](const uint16_t* W, int K, const uint16_t* x, const uint16_t* res, uint16_t* out) -> int {
    GemvParams p{};
    p.W = W; p.N = a.dim; p.K = K; p.x = x; p.ldx = K; p.ldo = a.dim;
    if (m->tp_size == 1) {
      p.out_bf16 = out; p.res = res;
      return launch_gemv<PRO_PLAIN, EPI_RESID>(L, mode, p, S, mb_rows);
    }
    int rc2;
    if (s->p2p_ready) {
      p.p2p = s->p2p; p.st = s->st;
      if ((rc2 = launch_gemv<PRO_PLAIN, EPI_P2P>(L, mode, p, S))) return rc2;
      return launch_kernel(L, p2p_reduce_resid_kernel, dim3(std::min(16, (S * a.dim + 255) / 256)), dim3(256), 0, s->p2p, s->st, res, out,
                           S * a.dim);
    }
    p.out_f32 = s->part;
    if ((rc2 = launch_gemv<PRO_PLAIN, EPI_F32RAW>(L, mode, p, S))) return rc2;
    NC(g_nccl.AllReduce(s->part, s->part, (size_t)S * a.dim, ncclFloat32_, ncclSum_, m->comm, s->stream));
    return launch_kernel(L, resid_from_f32_kernel, dim3(std::min(kWaveSMs, (S * a.dim + 255) / 256)), dim3(256), 0, (const float*)s->part,
                         res, out, (int64_t)S * a.dim);
  };
  for (int l = 0; l < n_layers; l++) {
    LayerW& W = m->layers[l];
    if ((rc = strict_scale(s->x, S))) return rc;
    {  // attn_norm -> wq|wk|wv -> RoPE -> KV append            (:222, :297-403)
      GemvParams p{};
      p.rscale = strict ? s->rs : nullptr;
      p.W = W.wqkv; p.N = m->q_l + 2 * m->kv_l; p.K = a.dim;
      p.x = s->x; p.ldx = a.dim; p.norm_w = W.attn_norm; p.eps = a.norm_eps;
      p.out_bf16 = s->q; p.ldo = m->q_l;
      p.q_dim = m->q_l; p.kv_dim = m->kv_l; p.head_dim = a.head_dim;
      p.cache_k = s->ck[l] + R.cache_off; p.cache_v = s->cv[l] + R.cache_off; p.cis = m->cis; p.pos_ptr = &s->st->pos;
      p.pos_arr = R.pos_arr; p.row_seq = R.row_seq; p.cache_seq_stride = R.seq_stride;
      if ((rc = launch_gemv<PRO_RMSNORM, EPI_QKV_ROPE>(L, mode, p, S, mb_rows))) return rc;
    }
    if ((rc = launch_attention(L, s, l, R, s->o, 0))) return rc;
    if ((rc = proj_resid(W.wo, m->q_l, s->o, s->x, s->h1))) return rc;            // wo + residual (:522, :232)
    if ((rc = strict_scale(s->h1, S))) return rc;
    {  // ffn_norm -> w1|w3 -> SiLU * up                             (:237, :601-614)
      GemvParams p{};
      p.rscale = strict ? s->rs : nullptr;
      p.W = W.w13; p.N = 2 * m->ffn_l; p.K = a.dim; p.x = s->h1; p.ldx = a.dim; p.norm_w = W.ffn_norm; p.eps = a.norm_eps;
      p.out_bf16 = s->mbuf; p.ldo = m->ffn_l; p.silu_tab = m->silu_tab;
      if ((rc = launch_gemv<PRO_RMSNORM, EPI_SWIGLU>(L, mode, p, S, mb_rows))) return rc;
    }
    if ((rc = proj_resid(W.w2, m->ffn_l, s->mbuf, s->h1, s->x))) return rc;        // w2 + residual (:619, :248)
  }
  if (R.head == HEAD_PER_ROW) return per_row_head(L, s, R);
  // output_norm -> output -> f32 logits (+ greedy argmax of the last row)   (:166-175; inference.go:207-216)
  const int rows = R.head_rows;
  const int row0 = S - rows;
  if ((rc = strict_scale(s->x + (size_t)row0 * a.dim, rows))) return rc;
  GemvParams p{};
  p.rscale = strict ? s->rs : nullptr;
  p.W = m->output; p.N = m->vocab_l; p.K = a.dim;
  p.x = s->x + (size_t)row0 * a.dim; p.ldx = a.dim; p.norm_w = m->norm; p.eps = a.norm_eps;
  p.out_f32 = R.head != HEAD_NONE ? s->logits : nullptr; p.ldo = m->vocab_l;
  p.n_offset = m->tp_rank * m->vocab_l;
  p.st = s->st; p.argmax_row = rows - 1; p.m_off = 0;
  p.publish = (m->tp_size == 1) ? 1 : 0;
  p.advance = R.advance ? 1 : 0; p.tok_out = s->d_tok_out;
  if ((rc = launch_gemv<PRO_RMSNORM, EPI_LOGITS>(L, mode, p, rows))) return rc;
  if (m->tp_size > 1) {
    if (s->p2p_ready) rc = launch_kernel(L, p2p_argmax_kernel, dim3(1), dim3(32), 0, s->p2p, s->st, R.advance ? 1 : 0, s->d_tok_out);
    else rc = reduce_argmax_publish(L, s, R.advance);
    if (rc) return rc;
    if (R.head != HEAD_NONE && R.gather && (rc = gather_logits(s, 0, rows))) return rc;
  }
  return 0;
}

// the tensor-core form of enqueue_forward (which routes here): projections as GEMMs, RoPE / KV append in rope_kv_kernel
static int enqueue_forward_tc(lnb_session* s, const Rows& R) {
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  const Launcher L{s->stream, LAUNCH_PDL, &s->launches};
  const int S = R.S;
  const int Mpad = (S + TC_BM - 1) / TC_BM * TC_BM;
  const int qkv_n = m->q_l + 2 * m->kv_l;
  int rc;
  if ((rc = launch_kernel(L, gather_rows_kernel, dim3(S), dim3(256), 0, (const uint16_t*)m->tok_embd, R.tokens, (const LnbDevState*)s->st,
                          s->x, a.dim)))
    return rc;
  const int n_layers = active_layers(s);
  const int ew_grid = m->sm_count * 8;
  // wo / w2 + residual: out = res + X W^T; tensor-parallel ranks sum their partials over NCCL first
  auto proj_resid = [&](const uint16_t* X8, const uint16_t* W, int K, const uint16_t* res, uint16_t* out) -> int {
    GemmTcParams g{};
    g.X8 = X8; g.W = W; g.M = S; g.N = a.dim; g.K = K; g.ldo = a.dim;
    if (m->tp_size == 1) {
      g.out_bf16 = out; g.res = res;
      return launch_gemm_tc<TC_EPI_RESID>(L, g);
    }
    g.out_f32 = s->part;
    if (int rc2 = launch_gemm_tc<TC_EPI_F32RAW>(L, g)) return rc2;
    NC(g_nccl.AllReduce(s->part, s->part, (size_t)S * a.dim, ncclFloat32_, ncclSum_, m->comm, s->stream));
    return launch_kernel(L, resid_from_f32_kernel, dim3(ew_grid), dim3(256), 0, (const float*)s->part, res, out, (int64_t)S * a.dim);
  };
  for (int l = 0; l < n_layers; l++) {
    LayerW& W = m->layers[l];
    if ((rc = launch_kernel(L, rmsnorm_x8_kernel, dim3(Mpad), dim3(256), 0, (const uint16_t*)s->x, a.dim, (const uint16_t*)W.attn_norm,
                            s->xn8, S, a.dim, a.norm_eps)))
      return rc;
    {
      GemmTcParams g{};
      g.X8 = s->xn8; g.W = W.wqkv; g.M = S; g.N = qkv_n; g.K = a.dim; g.out_bf16 = s->qkv_raw; g.ldo = qkv_n;
      if ((rc = launch_gemm_tc<TC_EPI_BF16>(L, g))) return rc;
    }
    if ((rc = launch_kernel(L, rope_kv_kernel, dim3(ew_grid), dim3(256), 0, (const uint16_t*)s->qkv_raw, qkv_n, s->q, m->q_l, m->kv_l,
                            a.head_dim, s->ck[l] + R.cache_off, s->cv[l] + R.cache_off, (const float*)m->cis, (const int32_t*)&s->st->pos, S,
                            R.pos_arr, R.row_seq, (long long)s->seq_len * m->kv_l)))
      return rc;
    if ((rc = launch_attention(L, s, l, R, s->o8, 1))) return rc;
    if ((rc = proj_resid(s->o8, W.wo, m->q_l, s->x, s->h1))) return rc;
    if ((rc = launch_kernel(L, rmsnorm_x8_kernel, dim3(Mpad), dim3(256), 0, (const uint16_t*)s->h1, a.dim, (const uint16_t*)W.ffn_norm,
                            s->xn8, S, a.dim, a.norm_eps)))
      return rc;
    {
      GemmTcParams g{};
      // SwiGLU in the epilogue: the hidden activations go straight into the X8 operand of the w2 GEMM
      g.X8 = s->xn8; g.W = W.w13; g.M = S; g.N = 2 * m->ffn_l; g.K = a.dim; g.out_bf16 = s->m8; g.ldo = m->ffn_l; g.silu_tab = m->silu_tab;
      if ((rc = launch_gemm_tc<TC_EPI_SWIGLU>(L, g))) return rc;
    }
    if ((rc = proj_resid(s->m8, W.w2, m->ffn_l, s->h1, s->x))) return rc;
  }
  // LM head: all rows on the tensor cores when asked for (and the vocabulary shard tiles), then the
  // last row through the GEMV, which also owns the greedy argmax (identical to the decode path)
  if (R.head == HEAD_PER_ROW) return per_row_head(L, s, R);
  if (R.head == HEAD_ALL && m->vocab_l % TC_BN == 0) {
    if ((rc = launch_kernel(L, rmsnorm_x8_kernel, dim3(Mpad), dim3(256), 0, (const uint16_t*)s->x, a.dim, (const uint16_t*)m->norm, s->xn8, S,
                            a.dim, a.norm_eps)))
      return rc;
    GemmTcParams g{};
    g.X8 = s->xn8; g.W = m->output; g.M = S - 1; g.N = m->vocab_l; g.K = a.dim; g.out_f32 = s->logits; g.ldo = m->vocab_l;
    if (S > 1 && (rc = launch_gemm_tc<TC_EPI_F32TRUNC>(L, g))) return rc;
  } else if (R.head == HEAD_ALL && S > 1) {
    GemvParams p{};
    p.W = m->output; p.N = m->vocab_l; p.K = a.dim; p.x = s->x; p.ldx = a.dim; p.norm_w = m->norm; p.eps = a.norm_eps;
    p.out_f32 = s->logits; p.ldo = m->vocab_l; p.st = nullptr; p.argmax_row = -1;
    if ((rc = launch_gemv<PRO_RMSNORM, EPI_LOGITS>(L, s->mode, p, S - 1))) return rc;
  }
  {
    GemvParams p{};
    p.W = m->output; p.N = m->vocab_l; p.K = a.dim;
    p.x = s->x + (size_t)(S - 1) * a.dim; p.ldx = a.dim; p.norm_w = m->norm; p.eps = a.norm_eps;
    p.out_f32 = R.head != HEAD_NONE ? s->logits + (R.head == HEAD_ALL ? (size_t)(S - 1) * m->vocab_l : 0) : nullptr;
    p.ldo = m->vocab_l; p.n_offset = m->tp_rank * m->vocab_l;
    p.st = s->st; p.argmax_row = 0; p.publish = (m->tp_size == 1) ? 1 : 0; p.advance = 0; p.tok_out = s->d_tok_out;
    if ((rc = launch_gemv<PRO_RMSNORM, EPI_LOGITS>(L, s->mode, p, 1))) return rc;
    if (m->tp_size > 1) {
      if ((rc = reduce_argmax_publish(L, s, false))) return rc;
      if (R.head != HEAD_NONE && R.gather && (rc = gather_logits(s, 0, R.head_rows))) return rc;
    }
  }
  return 0;
}

// ---- seeded sampling (sample.cuh, DESIGN.md §9b) ----------------------------------------------------------------
// both sampler kernels; each row is served by the one its parameters select (on the device: they may change between replays)
static int launch_sample_job(const Launcher& L, const SampleJob& J) {
  int rc = launch_kernel(L, sample_split_kernel, dim3((J.V + SMP_SLICE - 1) / SMP_SLICE, J.n), dim3(SMP_THREADS), 0, J);
  if (rc) return rc;
  return launch_kernel(L, sample_kernel, dim3(J.n), dim3(SMP_THREADS), 0, J);
}
// ---- penalties (penalty.cuh, DESIGN.md §9e) ---------------------------------------------------------------------------
static int launch_penalty_job(const Launcher& L, const PenaltyJob& J) {
  int rc = launch_kernel(L, penalty_count_kernel, dim3(PEN_COUNT_CTAS, J.n), dim3(PEN_THREADS), 0, J);
  if (rc) return rc;
  return launch_kernel(L, penalty_apply_kernel, dim3((J.V + PEN_SLICE - 1) / PEN_SLICE, J.n), dim3(PEN_THREADS), 0, J);
}

// One sampler launch over n rows of s->logits: row[i] of sequence seq[i] draws with p_next[i] (-1: st->pos, for a decode
// run whose step has advanced) into out[out_idx[i]]; decode: the token also feeds the next step (st->next_token) and
// lands in d_tok_out.  Only calls with a processed row launch it.  When a row is penalized, the penalty job first writes
// every row to d_pen_out (rows of other sequences unchanged) and the sampler reads them there; a penalized sequence that
// does not sample draws from the greedy slot d_samp[n_seq] (temperature 0: rank 0 of l').
static int launch_sample(lnb_session* s, int n, const int32_t* row, const int32_t* seq, const int32_t* p_next, const int32_t* out_idx,
                         int32_t* out, bool decode) {
  const Launcher L{s->stream, LAUNCH_PDL, &s->launches};
  const int V = s->m->a.vocab_size;
  SampleJob J{};
  J.logits = s->logits; J.ld = s->m->vocab_l; J.V = V; J.n = n;
  J.params = s->d_samp; J.wbuf = s->d_samp_w; J.pos_ptr = &s->st->pos; J.out = out;
  J.cand = s->d_samp_cand; J.cnt = reinterpret_cast<unsigned int*>(s->d_samp_cand + (size_t)s->samp_rows * SMP_MERGE);
  J.st = decode ? s->st : nullptr; J.tok_out = decode ? s->d_tok_out : nullptr;
  bool pen = false;
  for (int i = 0; i < n; i++) {
    J.row[i] = row[i]; J.slot[i] = s->samp_on[seq[i]] ? seq[i] : s->n_seq; J.p_next[i] = p_next[i]; J.out_idx[i] = out_idx ? out_idx[i] : 0;
    pen |= s->pen_on[seq[i]];
  }
  if (pen) {
    PenaltyJob P{};
    P.logits = s->logits; P.ld = s->m->vocab_l; P.V = V; P.n = n;
    P.params = s->d_pen; P.hist = s->d_hist; P.hist_len = s->seq_len;
    P.cnt = s->d_pen_cnt; P.out = s->d_pen_out; P.pos_ptr = &s->st->pos;
    for (int i = 0; i < n; i++) {
      P.row[i] = row[i]; P.slot[i] = seq[i]; P.seq[i] = seq[i]; P.p_next[i] = p_next[i]; P.on[i] = s->pen_on[seq[i]] ? 1 : 0;
      J.row[i] = i;
    }
    int rc = launch_penalty_job(L, P);
    if (rc) return rc;
    J.logits = s->d_pen_out; J.ld = V;
  }
  return launch_sample_job(L, J);
}

// ---- token log-probabilities (logprob.cuh, DESIGN.md §9d) -------------------------------------------------------------
static int launch_logprob_job(const Launcher& L, const LogprobJob& J, int n) {
  const dim3 grid((J.V + LP_SLICE - 1) / LP_SLICE, n);
  int rc = launch_kernel(L, logprob_rank_kernel, grid, dim3(LP_THREADS), 0, J);
  if (rc) return rc;
  return launch_kernel(L, logprob_mass_kernel, grid, dim3(LP_THREADS), 0, J);
}
// the job over rows d_lp_rows[0, n) (their table uploaded by lp_upload) of s->logits
static int launch_logprob(lnb_session* s, int n) {
  const int V = s->m->a.vocab_size, G = (V + LP_SLICE - 1) / LP_SLICE;
  LogprobJob J{};
  J.rows = s->d_lp_rows; J.top_n = s->d_lp_top; J.V = V;
  J.cand = s->d_lp_cand;
  J.above = reinterpret_cast<unsigned int*>(s->d_lp_cand + (size_t)s->lp_rows * G * LP_TOP);
  J.done = J.above + (size_t)s->lp_rows * G;
  return launch_logprob_job(Launcher{s->stream, LAUNCH_PDL, &s->launches}, J, n);
}
// row i of the next job: logits row `row` of s->logits, target *target, the record of sequence seq at position pos (+ *pos_ptr)
static void lp_row(lnb_session* s, int i, int row, const int32_t* target, int seq, int pos, const int32_t* pos_ptr) {
  LpRow& r = s->h_lp_rows[i];
  r.logits = s->logits + (size_t)row * s->m->vocab_l;
  r.target = target;
  r.rec = s->d_lp_rec + (size_t)seq * (s->seq_len + 1) + pos;
  r.rec_pos = pos_ptr;
  r.seq = seq;
  r.pad = 0;
}
// a written record -> its lnb_logprob (out zeroed by the caller)
static void lp_finish(const LpRecord& r, lnb_logprob* out) {
  const float m = lnb_logprob_key_logit(r.key[0]);
  out->token = r.target;
  out->rank = r.rank;
  out->logprob = lnb_logprob_finish(r.target_logit, m, r.sum);
  out->n_top = r.n_top;
  for (int j = 0; j < r.n_top; j++) {
    out->top_token[j] = lnb_logprob_key_index(r.key[j]);
    out->top_logprob[j] = lnb_logprob_finish(lnb_logprob_key_logit(r.key[j]), m, r.sum);
  }
}
static int lp_upload(lnb_session* s, int n) {
  CU(cudaMemcpyAsync(s->d_lp_rows, s->h_lp_rows, (size_t)n * sizeof(LpRow), cudaMemcpyHostToDevice, s->stream));
  return 0;
}

// The end of lnb_forward(_device), lnb_forward_batch, lnb_forward_ragged and lnb_forward_speculative.  Output row i is
// logits row row0 + i, of sequence seq[i] at next position p_next[i]; rows of processed sequences draw into samp_out[i], the
// greedy token of row i is at greedy[i].  Rows of sequences with logprobs on then write the record of p_next[i] for the
// token they emit.  host_logits (or NULL) gets logits rows [0, logits_rows), s->h_out[0, n) the tokens at d_tok (or NULL),
// then s->h_out[n] the sampled token of row 0 when the sampler writes beside them (samp_out != d_tok).
static int call_tail(lnb_session* s, int n, int row0, const int32_t* seq, const int32_t* p_next, int32_t* samp_out,
                     const int32_t* greedy, float* host_logits, int logits_rows, const int32_t* d_tok) {
  int32_t srow[8], sseq[8], spn[8], sidx[8];
  int ns = 0, nl = 0;
  for (int i = 0; i < n; i++)
    if (processed(s, seq[i])) { srow[ns] = row0 + i; sseq[ns] = seq[i]; spn[ns] = p_next[i]; sidx[ns] = i; ns++; }
  int rc;
  if (ns && (rc = launch_sample(s, ns, srow, sseq, spn, sidx, samp_out, false))) return rc;
  for (int i = 0; i < n; i++)
    if (s->lp_top[seq[i]] >= 0) lp_row(s, nl++, row0 + i, processed(s, seq[i]) ? samp_out + i : greedy + i, seq[i], p_next[i], nullptr);
  if (nl && ((rc = lp_upload(s, nl)) || (rc = launch_logprob(s, nl)))) return rc;
  lnb_model* m = s->m;
  if (host_logits) {
    const float* src = (m->tp_size > 1) ? s->logits_full : s->logits;
    CU(cudaMemcpyAsync(host_logits, src, (size_t)logits_rows * m->a.vocab_size * 4, cudaMemcpyDeviceToHost, s->stream));
  }
  if (d_tok) CU(cudaMemcpyAsync(s->h_out, d_tok, (size_t)n * 4, cudaMemcpyDeviceToHost, s->stream));
  if (d_tok && ns && samp_out != d_tok) CU(cudaMemcpyAsync(s->h_out + n, samp_out, 4, cudaMemcpyDeviceToHost, s->stream));
  if ((rc = p2p_err_enqueue(s))) return rc;
  if ((rc = sync_stream(s))) return rc;
  return p2p_err_check(s);
}

// The forward of lnb_forward and lnb_forward_device; the caller holds s->mu.  keep_logits: the logits of the last row, or
// of all S rows (all_rows), stay in s->logits.  host_logits: NULL, or where those rows are copied (tensor-parallel:
// gathered from the ranks first).  next_token: NULL, or receives the next token of the last row (greedy unless the active
// sequence samples); greedy_token: NULL, or receives the greedy token of the last row.  score (lnb_score, with all_rows):
// no token is emitted; row i writes the logprob record of position start_pos + 1 + i for the target d_lp_tgt[i].
static int forward_locked(lnb_session* s, const int32_t* tokens, int S, int start_pos, bool keep_logits, bool all_rows,
                          float* host_logits, int32_t* next_token, int32_t* greedy_token = nullptr, bool score = false) {
  if (!tokens) return fail(LNB_EINVAL, "NULL argument");
  if (S <= 0) return fail(LNB_EINVAL, "empty token array");  // llamatransformer.go:146-148
  if (S > s->max_rows) return fail(LNB_EINVAL, "S %d exceeds the session's max_rows %d", S, s->max_rows);
  if (start_pos < 0 || start_pos + S > s->seq_len)
    return fail(LNB_EINVAL, "positions [%d, %d) exceed SequenceLength %d", start_pos, start_pos + S, s->seq_len);
  if (S > 1 && start_pos != 0 && !s->allow_chunked)
    return fail(LNB_EINVAL, "S>1 requires startPos 0 (the reference's [S,S] mask does not broadcast to [S,T]); "
                "lnb_session_set_chunked_prefill enables the [S,T]-mask extension");
  for (int i = 0; i < S; i++)
    if (tokens[i] < 0 || tokens[i] >= s->m->a.vocab_size) return fail(LNB_EINVAL, "token id %d out of range", tokens[i]);
  lnb_model* m = s->m;
  CU(cudaSetDevice(m->device));
  s->kept_rows = 0;   // a logits handle is valid until the session's next forward (this call may overwrite or move them)
  const int32_t seq = s->active_seq, p_next = start_pos + S;
  const bool samp = processed(s, seq);   // the sampler and the logprob job read the last row's logits
  const int lrows = keep_logits ? (all_rows ? S : 1) : ((samp || s->lp_top[seq] >= 0) ? 1 : 0);
  int rc;
  if (lrows && (rc = ensure_logits(s, (size_t)(keep_logits && all_rows ? s->max_rows : 1)))) return rc;
  if (S == 1 && engine_ok(s)) {
    // decode step: ONE persistent kernel; the token id rides in the launch of set_state_kernel (4 bytes of kernel arguments)
    if ((rc = launch_record(s, rows_single(s, 1, nullptr, 0, false, false), tokens[0], start_pos))) return rc;
    if ((rc = enqueue_decode_engine(s, tokens[0], start_pos, 1, false, false, lrows ? s->logits : nullptr))) return rc;
    if (host_logits && (rc = gather_logits(s, 0, 1))) return rc;
  } else {
    memcpy(s->h_tok, tokens, (size_t)S * 4);
    CU(cudaMemcpyAsync(s->d_tokens, s->h_tok, (size_t)S * 4, cudaMemcpyHostToDevice, s->stream));
    if ((rc = set_state(s, start_pos, S, -1, false))) return rc;
    if ((rc = enqueue_forward(s, rows_single(s, S, s->d_tokens, lrows, false, host_logits != nullptr)))) return rc;
  }
  if (score) {
    for (int i = 0; i < S; i++) lp_row(s, i, i, s->d_lp_tgt + i, seq, start_pos + 1 + i, nullptr);
    if ((rc = lp_upload(s, S)) || (rc = launch_logprob(s, S))) return rc;
    return call_tail(s, 0, 0, &seq, &p_next, nullptr, nullptr, nullptr, 0, nullptr);
  }
  // the sampled token goes to d_samp_tok; st->next_token keeps the greedy one (lnb_session_logits_argmax)
  if ((rc = call_tail(s, 1, lrows - 1, &seq, &p_next, s->d_samp_tok, &s->st->next_token, host_logits, lrows,
                      (next_token || greedy_token) ? &s->st->next_token : nullptr)))
    return rc;
  if (next_token) *next_token = samp ? s->h_out[1] : s->h_out[0];
  if (greedy_token) *greedy_token = s->h_out[0];
  return 0;
}

extern "C" int lnb_forward(lnb_session* s, const int32_t* tokens, int S, int start_pos, float* logits, int all_rows,
                           int32_t* argmax_last) {
  if (!s) return fail(LNB_EINVAL, "NULL argument");
  std::lock_guard<std::mutex> lk(s->mu);
  return forward_locked(s, tokens, S, start_pos, logits != nullptr, all_rows != 0, logits, argmax_last);
}

// Forward whose logits stay on the device: the host mirror of LlamaTransformer.Forward hands the caller a tensor
// that carries a handle to them (ml.Tensor with a device view) and only lnb_session_logits_read copies rows out.
// inference.generateTokensInternal slices the last row and argmaxes it (inference.go:207-216): with the handle
// that is lnb_session_logits_argmax -- 4 bytes cross PCIe per token instead of S x 513 KB down and 513 KB up again.
// rows_kept: 1 = last row, S = all rows.  generation_out identifies the call (handles of older calls are stale).
extern "C" int lnb_forward_device(lnb_session* s, const int32_t* tokens, int S, int start_pos, int rows_kept,
                                  int32_t* argmax_last, int64_t* generation_out) {
  if (!s) return fail(LNB_EINVAL, "NULL argument");
  if (rows_kept != 1 && rows_kept != S) return fail(LNB_EINVAL, "rows_kept must be 1 or S");
  std::lock_guard<std::mutex> lk(s->mu);
  int32_t tok = -1, greedy = -1;
  const int rc = forward_locked(s, tokens, S, start_pos, true, rows_kept > 1, nullptr, &tok, &greedy);
  if (rc) return rc;
  if (argmax_last) *argmax_last = tok;
  s->kept_last_token = greedy;
  s->kept_rows = rows_kept;
  s->generation++;
  if (generation_out) *generation_out = s->generation;
  return 0;
}
static int logits_handle_check(lnb_session* s, int64_t generation, int row0, int rows) {
  if (generation != s->generation || s->kept_rows == 0)
    return fail(LNB_ESTATE, "logits handle of forward #%lld is stale (the session is at #%lld)", (long long)generation, (long long)s->generation);
  if (row0 < 0 || rows <= 0 || row0 + rows > s->kept_rows) return fail(LNB_EINVAL, "rows [%d, %d) outside the %d kept rows", row0, row0 + rows, s->kept_rows);
  return 0;
}
// rows [row0, row0+rows) of the kept logits -> host [rows, vocab] f32 (pinned staging; tensor-parallel: all-gather first,
// a collective -- every rank must make the same call)
extern "C" int lnb_session_logits_read(lnb_session* s, int64_t generation, int row0, int rows, float* host) {
  if (!s || !host) return fail(LNB_EINVAL, "NULL argument");
  std::lock_guard<std::mutex> lk(s->mu);
  int rc = logits_handle_check(s, generation, row0, rows);
  if (rc) return rc;
  lnb_model* m = s->m;
  CU(cudaSetDevice(m->device));
  const size_t V = (size_t)m->a.vocab_size, bytes = (size_t)rows * V * 4;
  const float* src = s->logits + (size_t)row0 * m->vocab_l;
  if (m->tp_size > 1) {
    if ((rc = gather_logits(s, row0, rows))) return rc;
    src = s->logits_full + (size_t)row0 * V;
  }
  if (bytes <= ((size_t)16 << 20)) {
    if (s->h_logits_bytes < bytes) {
      if (s->h_logits_pin) cudaFreeHost(s->h_logits_pin);
      s->h_logits_pin = nullptr; s->h_logits_bytes = 0;
      CU(cudaMallocHost((void**)&s->h_logits_pin, bytes));
      s->h_logits_bytes = bytes;
    }
    CU(cudaMemcpyAsync(s->h_logits_pin, src, bytes, cudaMemcpyDeviceToHost, s->stream));
    CU(cudaStreamSynchronize(s->stream));
    memcpy(host, s->h_logits_pin, bytes);
  } else {
    CU(cudaMemcpyAsync(host, src, bytes, cudaMemcpyDeviceToHost, s->stream));
    CU(cudaStreamSynchronize(s->stream));
  }
  return 0;
}
// ml.Argmax (operations_impl.go:513-548) of kept rows, on the device: first maximum wins, NaN never.  The last row's
// greedy token was already produced by the LM-head kernel of the forward (fused argmax) and is returned as is; other
// rows run argmax_f32_kernel on the kept logits (tensor-parallel: keys are max-reduced over the ranks, a collective).
__global__ void __launch_bounds__(256) argmax_key_rows_kernel(const float* __restrict__ x, int cols, int ld, int n_offset,
                                                              unsigned long long* __restrict__ keys) {
  __shared__ unsigned long long best[8];
  const float* xr = x + (size_t)blockIdx.x * ld;
  unsigned long long key = LNB_ARGMAX_EMPTY;
  for (int c = threadIdx.x; c < cols; c += 256) {
    const float v = xr[c];
    if (v > -3.402823466e+38f) {
      const unsigned long long k2 = argmax_key(v, (uint32_t)(c + n_offset));
      key = k2 > key ? k2 : key;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
    key = other > key ? other : key;
  }
  if ((threadIdx.x & 31) == 0) best[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; i++) key = best[i] > key ? best[i] : key;
    keys[blockIdx.x] = key;
  }
}
extern "C" int lnb_session_logits_argmax(lnb_session* s, int64_t generation, int row0, int rows, int32_t* out) {
  if (!s || !out) return fail(LNB_EINVAL, "NULL argument");
  std::lock_guard<std::mutex> lk(s->mu);
  int rc = logits_handle_check(s, generation, row0, rows);
  if (rc) return rc;
  lnb_model* m = s->m;
  CU(cudaSetDevice(m->device));
  if (rows == 1 && row0 + 1 == s->kept_rows) {   // the row the generate loop asks for: argmaxed by the forward itself
    out[0] = s->kept_last_token;
    return 0;
  }
  if (!s->d_keys) CU(cudaMalloc((void**)&s->d_keys, (size_t)s->max_rows * 8));
  unsigned long long* hk = reinterpret_cast<unsigned long long*>(s->h_err + 2);  // pinned, 8-byte aligned, 7 words free
  for (int r0 = 0; r0 < rows; r0 += 7) {
    const int n = rows - r0 < 7 ? rows - r0 : 7;
    argmax_key_rows_kernel<<<n, 256, 0, s->stream>>>(s->logits + (size_t)(row0 + r0) * m->vocab_l, m->vocab_l, m->vocab_l,
                                                      m->tp_rank * m->vocab_l, s->d_keys);
    s->launches++;
    if (m->tp_size > 1) NC(g_nccl.AllReduce(s->d_keys, s->d_keys, (size_t)n, ncclUint64_, ncclMax_, m->comm, s->stream));
    CU(cudaMemcpyAsync(hk, s->d_keys, (size_t)n * 8, cudaMemcpyDeviceToHost, s->stream));
    CU(cudaStreamSynchronize(s->stream));
    CU(cudaGetLastError());
    for (int i = 0; i < n; i++)
      out[r0 + i] = (hk[i] == LNB_ARGMAX_EMPTY) ? -1 : (int32_t)(0xffffffffu - (uint32_t)(hk[i] & 0xffffffffull));
  }
  return 0;
}

// ---- batched decode (BASELINE config 5: concurrent prompts) --------------------------------------
extern "C" int lnb_session_set_active_sequence(lnb_session* s, int seq) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  if (seq < 0 || seq >= s->n_seq) return fail(LNB_EINVAL, "sequence %d out of range (session has %d)", seq, s->n_seq);
  std::lock_guard<std::mutex> lk(s->mu);
  if (seq != s->active_seq) drop_graph(s);
  s->active_seq = seq;
  return 0;
}
// ---- seeded sampling: parameters of one sequence (sample.cuh, DESIGN.md §9b) ----------------------------------------
static int sampling_check(const lnb_sampling* p) {
  if (!std::isfinite(p->temperature) || p->temperature < 0.0f) return fail(LNB_EINVAL, "temperature %g must be finite and >= 0", (double)p->temperature);
  if (p->temperature == 0.0f) return 0;   // greedy: the other fields are unused
  if (p->top_k < 0) return fail(LNB_EINVAL, "top_k %d must be >= 0 (0: the whole vocabulary)", p->top_k);
  if (!(p->top_p > 0.0f && p->top_p <= 1.0f)) return fail(LNB_EINVAL, "top_p %g must be in (0, 1]", (double)p->top_p);
  return 0;
}
// The sampler's buffers, allocated by the first sampler set or penalty enable: n_seq parameter slots plus the greedy slot
// d_samp[n_seq] (zeroed: temperature 0) of penalized sequences that do not sample, weights of n_seq rows, one token; all or
// nothing
static int samp_alloc(lnb_session* s) {
  if (s->d_samp) return 0;
  const size_t b_par = (size_t)(s->n_seq + 1) * sizeof(lnb_sampling), b_w = (size_t)s->n_seq * s->m->a.vocab_size * 8;
  const size_t b_cand = (size_t)s->n_seq * (SMP_MERGE * 8 + 4);
  lnb_sampling* d_par = nullptr;
  unsigned long long *d_w = nullptr, *d_cand = nullptr;
  int32_t* d_tok = nullptr;
  cudaError_t e = cudaMalloc((void**)&d_par, b_par);
  if (e == cudaSuccess) e = cudaMalloc((void**)&d_w, b_w);
  if (e == cudaSuccess) e = cudaMalloc((void**)&d_tok, 16);
  if (e == cudaSuccess) e = cudaMalloc((void**)&d_cand, b_cand);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_par, 0, b_par, s->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_cand, 0, b_cand, s->stream);   // the split sampler's counters start at 0
  if (e != cudaSuccess) {
    cudaGetLastError();
    cudaStreamSynchronize(s->stream);
    cudaFree(d_par); cudaFree(d_w); cudaFree(d_tok); cudaFree(d_cand);
    cudaGetLastError();
    return fail(LNB_ENOMEM, "sampler buffers: %zu bytes of device memory asked for: %s", b_par + b_w + 16 + b_cand, cudaGetErrorString(e));
  }
  s->d_samp = d_par; s->d_samp_w = d_w; s->d_samp_tok = d_tok; s->d_samp_cand = d_cand;
  s->samp_rows = s->n_seq;
  return 0;
}
extern "C" int lnb_session_set_sampling(lnb_session* s, int seq, const lnb_sampling* p) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  if (seq < 0 || seq >= s->n_seq) return fail(LNB_EINVAL, "sequence %d out of range (session has %d)", seq, s->n_seq);
  if (s->m->tp_size > 1)
    return fail(LNB_EINVAL, "sampling is not built for tensor parallelism (tp_size %d: the logits are sharded over the vocabulary)", s->m->tp_size);
  int rc;
  if (p && (rc = sampling_check(p))) return rc;
  const bool on = p && p->temperature > 0.0f;
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(s->m->device));
  if (on && (rc = samp_alloc(s))) return rc;
  if (on) {   // stream-ordered, no host synchronisation; a captured decode graph reads the slot when it replays
    sample_set_params_kernel<<<1, 1, 0, s->stream>>>(s->d_samp + seq, *p);
    CU(cudaGetLastError());
  }
  s->samp_on[seq] = on;
  return 0;
}

// ---- penalties: parameters of one sequence and its token history (penalty.cuh, DESIGN.md §9e) --------------------------
static int penalties_check(const lnb_penalties* p, int V) {
  if (!std::isfinite(p->repetition_penalty) || !(p->repetition_penalty > 0.0f))
    return fail(LNB_EINVAL, "repetition_penalty %g must be finite and > 0", (double)p->repetition_penalty);
  if (!std::isfinite(p->frequency_penalty)) return fail(LNB_EINVAL, "frequency_penalty %g must be finite", (double)p->frequency_penalty);
  if (!std::isfinite(p->presence_penalty)) return fail(LNB_EINVAL, "presence_penalty %g must be finite", (double)p->presence_penalty);
  if (p->window < 0) return fail(LNB_EINVAL, "window %d must be >= 0 (0: every position)", p->window);
  if (p->first_pos < 0) return fail(LNB_EINVAL, "first_pos %d must be >= 0", p->first_pos);
  if (p->n_bias < 0 || p->n_bias > LNB_LOGIT_BIAS_MAX) return fail(LNB_EINVAL, "n_bias %d must be in [0, %d]", p->n_bias, LNB_LOGIT_BIAS_MAX);
  for (int j = 0; j < p->n_bias; j++) {
    const int t = p->bias_token[j];
    if (t < 0 || t >= V) return fail(LNB_EINVAL, "bias_token[%d] = %d outside [0, %d)", j, t, V);
    for (int k = 0; k < j; k++)
      if (p->bias_token[k] == t) return fail(LNB_EINVAL, "bias_token[%d] = %d repeats bias_token[%d]", j, t, k);
    const float b = p->bias[j];
    if (!(std::isfinite(b) || b == -INFINITY)) return fail(LNB_EINVAL, "bias[%d] = %g must be finite or -inf", j, (double)b);
  }
  return 0;
}
extern "C" int lnb_session_set_penalties(lnb_session* s, int seq, const lnb_penalties* p) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  if (seq < 0 || seq >= s->n_seq) return fail(LNB_EINVAL, "sequence %d out of range (session has %d)", seq, s->n_seq);
  if (s->m->tp_size > 1)
    return fail(LNB_EINVAL, "penalties are not built for tensor parallelism (tp_size %d: the logits are sharded over the vocabulary)", s->m->tp_size);
  const int V = s->m->a.vocab_size;
  int rc;
  if (p && (rc = penalties_check(p, V))) return rc;
  const bool on = p && !lnb_pen_neutral(p);
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(s->m->device));
  if (on && !s->d_hist) {   // history of every sequence and position, parameter slots, the job's scratch; all or nothing
    const size_t b_hist = (size_t)s->n_seq * s->seq_len * 4, b_par = (size_t)s->n_seq * sizeof(lnb_penalties),
                 b_cnt = (size_t)PEN_MAX_ROWS * V * 4, b_out = (size_t)PEN_MAX_ROWS * V * 4;
    int32_t* d_hist = nullptr;
    lnb_penalties* d_par = nullptr;
    unsigned int* d_cnt = nullptr;
    float* d_out = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_hist, b_hist);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_par, b_par);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_cnt, b_cnt);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_out, b_out);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_hist, 0xff, b_hist, s->stream);   // -1: no token recorded
    if (e == cudaSuccess) e = cudaMemsetAsync(d_cnt, 0, b_cnt, s->stream);        // the counts start at 0
    if (e != cudaSuccess) {
      cudaGetLastError();
      cudaStreamSynchronize(s->stream);
      cudaFree(d_hist); cudaFree(d_par); cudaFree(d_cnt); cudaFree(d_out);
      cudaGetLastError();
      return fail(LNB_ENOMEM, "penalty history and scratch: %zu bytes of device memory asked for (history %zu): %s",
                  b_hist + b_par + b_cnt + b_out, b_hist, cudaGetErrorString(e));
    }
    if ((rc = samp_alloc(s))) {   // the sampler draws every penalized token
      cudaStreamSynchronize(s->stream);
      cudaFree(d_hist); cudaFree(d_par); cudaFree(d_cnt); cudaFree(d_out);
      return rc;
    }
    s->d_hist = d_hist; s->d_pen = d_par; s->d_pen_cnt = d_cnt; s->d_pen_out = d_out;
  } else if (on && (rc = samp_alloc(s))) {
    return rc;
  }
  if (on) {   // stream-ordered, no host synchronisation; a captured decode graph reads the slot when it replays
    if (!s->pen_on[seq]) CU(cudaMemsetAsync(s->d_hist + (size_t)seq * s->seq_len, 0xff, (size_t)s->seq_len * 4, s->stream));
    penalty_set_params_kernel<<<1, 1, 0, s->stream>>>(s->d_pen + seq, *p);
    CU(cudaGetLastError());
  }
  s->pen_on[seq] = on;
  return 0;
}

// ---- token log-probabilities: records, switches and scoring (logprob.cuh, DESIGN.md §9d) ------------------------------
extern "C" int lnb_session_set_logprobs(lnb_session* s, int seq, int top_n) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  if (seq < 0 || seq >= s->n_seq) return fail(LNB_EINVAL, "sequence %d out of range (session has %d)", seq, s->n_seq);
  if (top_n < -1 || top_n > LNB_LOGPROBS_TOP_MAX) return fail(LNB_EINVAL, "top_n %d must be in [-1, %d] (-1: off)", top_n, LNB_LOGPROBS_TOP_MAX);
  if (s->m->tp_size > 1)
    return fail(LNB_EINVAL, "logprobs are not built for tensor parallelism (tp_size %d: the logits are sharded over the vocabulary)", s->m->tp_size);
  const int V = s->m->a.vocab_size;
  if (V > LP_MAX_VOCAB) return fail(LNB_EINVAL, "logprobs serve vocabularies of up to %d tokens (this model has %d)", LP_MAX_VOCAB, V);
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(s->m->device));
  if (top_n >= 0 && !s->d_lp_rec) {   // records of every sequence and position, the job's table and scratch; all or nothing
    const int rows = std::max(s->max_rows, 8), G = (V + LP_SLICE - 1) / LP_SLICE;
    const size_t b_rec = (size_t)s->n_seq * (s->seq_len + 1) * sizeof(LpRecord), b_top = (size_t)s->n_seq * 4,
                 b_tgt = (size_t)s->max_rows * 4, b_rows = (size_t)rows * sizeof(LpRow),
                 b_cand = (size_t)rows * G * (LP_TOP * 8 + 4) + (size_t)rows * 4;
    LpRecord* d_rec = nullptr;
    int32_t *d_top = nullptr, *d_tgt = nullptr;
    LpRow *d_rows = nullptr, *h_rows = nullptr;
    unsigned long long* d_cand = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_rec, b_rec);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_top, b_top);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_tgt, b_tgt);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_rows, b_rows);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_cand, b_cand);
    if (e == cudaSuccess) e = cudaMallocHost((void**)&h_rows, b_rows);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_rec, 0xff, b_rec, s->stream);   // target -1: never written
    if (e == cudaSuccess) e = cudaMemsetAsync(d_top, 0xff, b_top, s->stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_cand, 0, b_cand, s->stream);     // the merge counters start at 0
    if (e != cudaSuccess) {
      cudaGetLastError();
      cudaStreamSynchronize(s->stream);
      cudaFree(d_rec); cudaFree(d_top); cudaFree(d_tgt); cudaFree(d_rows); cudaFree(d_cand);
      if (h_rows) cudaFreeHost(h_rows);
      cudaGetLastError();
      return fail(LNB_ENOMEM, "logprob records and scratch: %zu bytes of device memory asked for (records %zu): %s",
                  b_rec + b_top + b_tgt + b_rows + b_cand, b_rec, cudaGetErrorString(e));
    }
    s->d_lp_rec = d_rec; s->d_lp_top = d_top; s->d_lp_tgt = d_tgt; s->d_lp_rows = d_rows; s->d_lp_cand = d_cand; s->h_lp_rows = h_rows;
    s->lp_rows = rows;
  }
  if (s->d_lp_top) {   // stream-ordered; a captured decode graph reads the slot when it replays
    if (top_n >= 0 || s->lp_top[seq] >= 0) {
      logprob_set_top_n_kernel<<<1, 1, 0, s->stream>>>(s->d_lp_top + seq, top_n);
      CU(cudaGetLastError());
    }
  }
  s->lp_top[seq] = top_n;
  return 0;
}

extern "C" int lnb_session_logprobs_read(lnb_session* s, int seq, int pos0, int n, lnb_logprob* out) {
  if (!s || !out) return fail(LNB_EINVAL, "NULL argument");
  if (seq < 0 || seq >= s->n_seq) return fail(LNB_EINVAL, "sequence %d out of range (session has %d)", seq, s->n_seq);
  if (n < 1 || pos0 < 1 || (int64_t)pos0 + n - 1 > s->seq_len)
    return fail(LNB_EINVAL, "positions [%d, %lld) outside [1, %d]", pos0, (long long)pos0 + n, s->seq_len);
  std::lock_guard<std::mutex> lk(s->mu);
  memset(out, 0, (size_t)n * sizeof(lnb_logprob));
  for (int i = 0; i < n; i++) out[i].token = -1;
  if (!s->d_lp_rec) return 0;   // logprobs were never on: nothing was written
  CU(cudaSetDevice(s->m->device));
  std::vector<LpRecord> rec((size_t)n);
  CU(cudaMemcpyAsync(rec.data(), s->d_lp_rec + (size_t)seq * (s->seq_len + 1) + pos0, (size_t)n * sizeof(LpRecord),
                     cudaMemcpyDeviceToHost, s->stream));
  CU(cudaStreamSynchronize(s->stream));
  for (int i = 0; i < n; i++)
    if (rec[i].target >= 0) lp_finish(rec[i], out + i);
  return 0;
}

extern "C" int lnb_score(lnb_session* s, const int32_t* tokens, int n, int start_pos) {
  if (!s || !tokens) return fail(LNB_EINVAL, "NULL argument");
  if (n < 2 || n - 1 > s->max_rows) return fail(LNB_EINVAL, "n %d must be in [2, max_rows + 1 = %d]", n, s->max_rows + 1);
  if (tokens[n - 1] < 0 || tokens[n - 1] >= s->m->a.vocab_size) return fail(LNB_EINVAL, "token id %d out of range", tokens[n - 1]);
  std::lock_guard<std::mutex> lk(s->mu);
  if (s->lp_top[s->active_seq] < 0)
    return fail(LNB_ESTATE, "sequence %d has logprobs off (lnb_session_set_logprobs)", s->active_seq);
  CU(cudaSetDevice(s->m->device));
  // the targets, stream-ordered before the job: staged in the pinned h_tok words [max_rows, 2 max_rows), beside the forward's
  // token ids [0, n - 1); no earlier call still reads them (every call synchronises its stream before it returns)
  int32_t* h_tgt = s->h_tok + s->max_rows;
  memcpy(h_tgt, tokens + 1, (size_t)(n - 1) * 4);
  CU(cudaMemcpyAsync(s->d_lp_tgt, h_tgt, (size_t)(n - 1) * 4, cudaMemcpyHostToDevice, s->stream));
  return forward_locked(s, tokens, n - 1, start_pos, true, true, nullptr, nullptr, nullptr, true);
}

// ---- fork / permute sequences (seqcopy.cuh, DESIGN.md §9f) -------------------------------------------------------------
// ONE stream-ordered launch: positions [pos0, pos1) of sequence dst[i] get what sequence src[i] held there before the call,
// in K and V of every layer, the penalty history and the logprob records (the last two when allocated).  Sampler and
// penalty parameters stay with their slot; the active sequence, a logits handle and a captured decode graph are untouched.
extern "C" int lnb_session_copy_sequences(lnb_session* s, int n, const int32_t* src, const int32_t* dst, int pos0, int pos1) {
  if (!s || !src || !dst) return fail(LNB_EINVAL, "NULL argument");
  lnb_model* m = s->m;
  if (m->tp_size > 1) return fail(LNB_EINVAL, "copying sequences is not built for tensor parallelism (tp_size %d)", m->tp_size);
  if (n < 1 || n > s->n_seq) return fail(LNB_EINVAL, "n %d must be in [1, n_seq = %d]", n, s->n_seq);
  for (int i = 0; i < n; i++) {
    if (src[i] < 0 || src[i] >= s->n_seq) return fail(LNB_EINVAL, "src[%d] = %d outside [0, %d)", i, src[i], s->n_seq);
    if (dst[i] < 0 || dst[i] >= s->n_seq) return fail(LNB_EINVAL, "dst[%d] = %d outside [0, %d)", i, dst[i], s->n_seq);
    for (int j = 0; j < i; j++)
      if (dst[j] == dst[i]) return fail(LNB_EINVAL, "dst[%d] = %d repeats dst[%d]", i, dst[i], j);
  }
  if (pos0 < 0 || pos0 >= pos1 || pos1 > s->seq_len)
    return fail(LNB_EINVAL, "positions [%d, %d) must satisfy 0 <= pos0 < pos1 <= seq_len = %d", pos0, pos1, s->seq_len);
  const int L = m->a.n_layers;
  if (L > SC_MAX_LAYERS) return fail(LNB_EINVAL, "copying sequences serves up to %d layers (this model has %d)", SC_MAX_LAYERS, L);
  static_assert(sizeof(LpRecord) % 16 == 0, "records move as 16-byte vectors");
  // cache rows move as 16-byte vectors too: kv_l * 2 bytes must be a multiple of 16 (model creation makes kv_l a multiple of 32)
  if ((m->kv_l * 2) % 16) return fail(LNB_EINVAL, "cache rows of %d bytes are not a multiple of 16", m->kv_l * 2);
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(m->device));
  const long long row16 = (long long)m->kv_l * 2 / 16, rec16 = (long long)sizeof(LpRecord) / 16, np = pos1 - pos0;
  SeqCopyJob J{};
  J.n = n;
  for (int i = 0; i < n; i++) { J.src[i] = src[i]; J.dst[i] = dst[i]; }
  J.n_kv = 2 * L;
  J.kv_stride = (long long)s->seq_len * row16; J.kv_len = np * row16;
  J.kv_tiles = (J.kv_len + SC_TILE - 1) / SC_TILE;
  for (int l = 0; l < L; l++) {
    J.kv[l] = reinterpret_cast<uint4*>(s->ck[l]) + pos0 * row16;
    J.kv[L + l] = reinterpret_cast<uint4*>(s->cv[l]) + pos0 * row16;
  }
  if (s->d_lp_rec) {
    J.rec = reinterpret_cast<uint4*>(s->d_lp_rec + pos0);
    J.rec_stride = (long long)(s->seq_len + 1) * rec16; J.rec_len = np * rec16;
    J.rec_tiles = (J.rec_len + SC_TILE - 1) / SC_TILE;
  }
  long long hist_tiles = 0;
  if (s->d_hist) {
    J.hist = s->d_hist + pos0;
    J.hist_stride = s->seq_len; J.hist_len = np;
    hist_tiles = (J.hist_len + SC_TILE - 1) / SC_TILE;
  }
  const long long grid = (long long)J.n_kv * J.kv_tiles + J.rec_tiles + hist_tiles;
  if (grid > 0x7fffffffLL) return fail(LNB_EINVAL, "%lld tiles exceed one grid", grid);
  return launch_kernel(Launcher{s->stream, LAUNCH_PDL, &s->launches}, seqcopy_kernel, dim3((unsigned)grid), dim3(SC_THREADS), 0, J);
}

// One decode step for n independent sequences (rows 0..n-1 = sequences 0..n-1): tokens[i] is fed at
// positions[i] of sequence i.  The weights are streamed ONCE for all rows (the reference would run n
// separate Forward calls on n InferenceContexts, SURVEY F10; every row sees exactly the arithmetic of its
// own S=1 Forward).  logits: NULL or host [n, vocab] f32; argmax_out[n] = greedy token per sequence.
extern "C" int lnb_forward_batch(lnb_session* s, const int32_t* tokens, const int32_t* positions, int n, float* logits,
                                 int32_t* argmax_out) {
  if (!s || !tokens || !positions) return fail(LNB_EINVAL, "NULL argument");
  if (n < 1 || n > s->n_seq) return fail(LNB_EINVAL, "n %d exceeds the session's %d sequences", n, s->n_seq);
  for (int i = 0; i < n; i++) {
    if (tokens[i] < 0 || tokens[i] >= s->m->a.vocab_size) return fail(LNB_EINVAL, "token id %d out of range", tokens[i]);
    if (positions[i] < 0 || positions[i] >= s->seq_len) return fail(LNB_EINVAL, "position %d exceeds SequenceLength %d", positions[i], s->seq_len);
  }
  std::lock_guard<std::mutex> lk(s->mu);
  lnb_model* m = s->m;
  CU(cudaSetDevice(m->device));
  s->kept_rows = 0;   // a logits handle is valid until the session's next forward (this call may overwrite or move them)
  int rc = ensure_logits(s, (size_t)s->max_rows);
  if (rc) return rc;
  memcpy(s->h_tok, tokens, (size_t)n * 4);
  memcpy(s->h_pos, positions, (size_t)n * 4);
  CU(cudaMemcpyAsync(s->d_tokens, s->h_tok, (size_t)n * 4, cudaMemcpyHostToDevice, s->stream));
  CU(cudaMemcpyAsync(s->d_pos_arr, s->h_pos, (size_t)n * 4, cudaMemcpyHostToDevice, s->stream));
  int32_t seq[8], p_next[8];
  bool samp = false;   // a row is processed or has logprobs on: the engine stores the logits
  for (int i = 0; i < n; i++) { seq[i] = i; p_next[i] = positions[i] + 1; samp |= processed(s, i) || s->lp_top[i] >= 0; }
  if (batch_engine_ok(s)) {
    // ONE launch of the batch engine: every weight matrix streamed once for all n sequences
    if ((rc = launch_record(s, rows_batch(s, n)))) return rc;
    if ((rc = batch_engine_build(s, (logits || samp) ? s->logits : nullptr))) return rc;
    if ((rc = batch_engine_launch(s, n, s->d_tokens, s->d_pos_arr, nullptr))) return rc;
    if (logits && (rc = gather_logits(s, 0, n))) return rc;
  } else {
    if (!s->sdpa_smem_decode && !s->ss.sc)
      return fail(LNB_EINVAL, "batched decode beyond the shared-memory attention kernel needs head_dim <= 128 and n_rep <= 8");
    if ((rc = set_state(s, 0, n, -1, false))) return rc;
    if ((rc = enqueue_forward(s, rows_batch(s, n)))) return rc;
  }
  if ((rc = call_tail(s, n, 0, seq, p_next, s->d_next_arr, s->d_next_arr, logits, n, argmax_out ? s->d_next_arr : nullptr))) return rc;
  if (argmax_out) memcpy(argmax_out, s->h_out, (size_t)n * 4);
  return 0;
}

// ---- ragged calls (continuous batching): segments of several sequences at their own positions in ONE forward ----------
// Buffers of the first ragged call: the row map on the device and, when the session has none or a smaller one,
// stream-attention scratch for max_rows rows per launch group.  Nothing is replaced unless every allocation succeeded, so a
// failure (LNB_ENOMEM) leaves the session as it was.
static int ragged_alloc(lnb_session* s) {
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  const size_t words = row_map_words(s->max_rows);
  SsScratch x{};
  size_t sc_b, z_b, op_b;
  ss_plan(x, s->seq_len, s->max_rows, m->q_l / a.head_dim, a.head_dim, &sc_b, &z_b, &op_b);
  const bool need_ss = !s->ss.sc || s->ss.rows < x.rows;
  if (s->d_rag && !need_ss) return 0;
  const size_t asked = (s->d_rag ? 0 : words * 4) + (need_ss ? sc_b + z_b + op_b : 0);
  int32_t* d_rag = nullptr;
  cudaError_t e = cudaSuccess;
  if (!s->d_rag) e = cudaMalloc((void**)&d_rag, words * 4);
  if (e == cudaSuccess && need_ss) e = cudaMalloc((void**)&x.sc, sc_b);
  if (e == cudaSuccess && need_ss) e = cudaMalloc((void**)&x.z, z_b);
  if (e == cudaSuccess && need_ss) e = cudaMalloc((void**)&x.op, op_b);
  if (e != cudaSuccess) {
    cudaGetLastError();
    cudaFree(d_rag); cudaFree(x.sc); cudaFree(x.z); cudaFree(x.op);
    cudaGetLastError();
    return fail(LNB_ENOMEM, "ragged-call buffers: %zu bytes of device memory asked for (stream-attention scratch for %d rows: %zu): %s", asked,
                x.rows, need_ss ? sc_b + z_b + op_b : (size_t)0, cudaGetErrorString(e));
  }
  if (d_rag) s->d_rag = d_rag;
  if (need_ss) {
    CU(cudaStreamSynchronize(s->stream));   // batched steps may still read the old scratch
    cudaFree(s->ss.sc); cudaFree(s->ss.z); cudaFree(s->ss.op);
    s->ss = x;
  }
  return 0;
}

extern "C" int lnb_forward_ragged(lnb_session* s, int n_segs, const int32_t* seq, const int32_t* start_pos, const int32_t* len,
                                  const int32_t* tokens, float* logits, int32_t* argmax_out) {
  if (!s || !seq || !start_pos || !len || !tokens) return fail(LNB_EINVAL, "NULL argument");
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  if (m->tp_size > 1) return fail(LNB_EINVAL, "lnb_forward_ragged is not built for tensor parallelism (tp_size %d)", m->tp_size);
  if (!ss_shape_ok(a.head_dim, a.n_heads / a.n_kv_heads))
    return fail(LNB_EINVAL, "ragged calls run the streamed attention kernels, which serve head_dim <= 128 and n_rep <= 8");
  if (n_segs < 1 || n_segs > s->n_seq) return fail(LNB_EINVAL, "n_segs %d must be in [1, %d] (the session's sequences)", n_segs, s->n_seq);
  bool used[8] = {false, false, false, false, false, false, false, false};
  int64_t rows64 = 0;
  for (int i = 0; i < n_segs; i++) {
    if (seq[i] < 0 || seq[i] >= s->n_seq) return fail(LNB_EINVAL, "segment %d: sequence %d out of range (session has %d)", i, seq[i], s->n_seq);
    if (used[seq[i]]) return fail(LNB_EINVAL, "segment %d: sequence %d has a segment already (one per sequence per call)", i, seq[i]);
    used[seq[i]] = true;
    if (len[i] < 1) return fail(LNB_EINVAL, "segment %d: len %d must be >= 1", i, len[i]);
    if (start_pos[i] < 0 || (int64_t)start_pos[i] + len[i] > s->seq_len)
      return fail(LNB_EINVAL, "segment %d: positions [%d, %lld) exceed SequenceLength %d", i, start_pos[i], (long long)start_pos[i] + len[i],
                  s->seq_len);
    rows64 += len[i];
  }
  if (rows64 > s->max_rows) return fail(LNB_EINVAL, "the segments carry %lld rows, more than the session's max_rows %d", (long long)rows64, s->max_rows);
  const int rows = (int)rows64;
  for (int r = 0; r < rows; r++)
    if (tokens[r] < 0 || tokens[r] >= a.vocab_size) return fail(LNB_EINVAL, "token id %d (row %d) out of range", tokens[r], r);
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(m->device));
  int rc;
  if ((rc = ragged_alloc(s))) return rc;
  if ((rc = ensure_logits(s, (size_t)n_segs))) return rc;
  s->kept_rows = 0;   // a logits handle is valid until the session's next forward
  // [tokens | row_seq | row_pos | last row of each segment]: one pinned staging copy
  int32_t* h = s->h_tok;
  memcpy(h, tokens, (size_t)rows * 4);
  for (int i = 0, r = 0; i < n_segs; i++) {
    for (int k = 0; k < len[i]; k++, r++) {
      h[rows + r] = seq[i];
      h[2 * rows + r] = start_pos[i] + k;
    }
    h[3 * rows + i] = r - 1;
  }
  CU(cudaMemcpyAsync(s->d_rag, h, (size_t)(3 * rows + n_segs) * 4, cudaMemcpyHostToDevice, s->stream));
  bool pen = false;
  for (int i = 0; i < n_segs; i++) pen |= s->pen_on[seq[i]];
  if ((rc = enqueue_forward(s, rows_ragged(s, rows, n_segs, pen)))) return rc;
  int32_t p_next[8];
  for (int i = 0; i < n_segs; i++) p_next[i] = start_pos[i] + len[i];
  if ((rc = call_tail(s, n_segs, 0, seq, p_next, s->d_next_arr, s->d_next_arr, logits, n_segs, argmax_out ? s->d_next_arr : nullptr))) return rc;
  if (argmax_out) memcpy(argmax_out, s->h_out, (size_t)n_segs * 4);
  return 0;
}

// ---- speculative verification: a sequence's last emitted token and k drafted tokens as k + 1 rows of ONE forward -------
// Sampler scratch for one launch of `rows` rows (a speculative call may draw up to 8 rows of one sequence, more than the
// session has sequences).  Nothing is replaced unless every allocation succeeded.  A captured decode graph that ends in the
// sampler holds the old scratch: it is dropped and re-captured by the next lnb_decode_run.
static int samp_grow(lnb_session* s, int rows) {
  if (s->samp_rows >= rows) return 0;
  const size_t b_w = (size_t)rows * s->m->a.vocab_size * 8, b_cand = (size_t)rows * (SMP_MERGE * 8 + 4);
  unsigned long long *d_w = nullptr, *d_cand = nullptr;
  cudaError_t e = cudaMalloc((void**)&d_w, b_w);
  if (e == cudaSuccess) e = cudaMalloc((void**)&d_cand, b_cand);
  if (e == cudaSuccess) e = cudaMemsetAsync(d_cand, 0, b_cand, s->stream);   // the split sampler's counters start at 0
  if (e != cudaSuccess) {
    cudaGetLastError();
    cudaFree(d_w); cudaFree(d_cand);
    cudaGetLastError();
    return fail(LNB_ENOMEM, "sampler scratch for %d rows: %zu bytes of device memory asked for: %s", rows, b_w + b_cand, cudaGetErrorString(e));
  }
  if (s->graph_sampled) drop_graph(s);
  CU(cudaStreamSynchronize(s->stream));   // earlier sampler launches may still use the old scratch
  cudaFree(s->d_samp_w); cudaFree(s->d_samp_cand);
  s->d_samp_w = d_w; s->d_samp_cand = d_cand; s->samp_rows = rows;
  return 0;
}

extern "C" int lnb_forward_speculative(lnb_session* s, int n_segs, const int32_t* seq, const int32_t* start_pos, const int32_t* n_draft,
                                       const int32_t* tokens, float* logits, int32_t* next_out, int32_t* n_accepted) {
  if (!s || !seq || !start_pos || !n_draft || !tokens) return fail(LNB_EINVAL, "NULL argument");
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  if (m->tp_size > 1) return fail(LNB_EINVAL, "lnb_forward_speculative is not built for tensor parallelism (tp_size %d)", m->tp_size);
  if (n_segs < 1 || n_segs > s->n_seq) return fail(LNB_EINVAL, "n_segs %d must be in [1, %d] (the session's sequences)", n_segs, s->n_seq);
  const int budget = std::min(8, s->max_rows);
  bool used[8] = {false, false, false, false, false, false, false, false};
  int64_t rows64 = 0;
  for (int i = 0; i < n_segs; i++) {
    if (seq[i] < 0 || seq[i] >= s->n_seq) return fail(LNB_EINVAL, "segment %d: sequence %d out of range (session has %d)", i, seq[i], s->n_seq);
    if (used[seq[i]]) return fail(LNB_EINVAL, "segment %d: sequence %d has a segment already (one per sequence per call)", i, seq[i]);
    used[seq[i]] = true;
    if (n_draft[i] < 0) return fail(LNB_EINVAL, "segment %d: n_draft %d must be >= 0", i, n_draft[i]);
    if (start_pos[i] < 0 || (int64_t)start_pos[i] + n_draft[i] >= s->seq_len)
      return fail(LNB_EINVAL, "segment %d: positions [%d, %lld] exceed SequenceLength %d", i, start_pos[i],
                  (long long)start_pos[i] + n_draft[i], s->seq_len);
    rows64 += 1 + (int64_t)n_draft[i];
  }
  if (rows64 > budget)
    return fail(LNB_EINVAL, "the segments carry %lld rows, more than min(8, max_rows) = %d", (long long)rows64, budget);
  const int rows = (int)rows64;
  for (int r = 0; r < rows; r++)
    if (tokens[r] < 0 || tokens[r] >= a.vocab_size) return fail(LNB_EINVAL, "token id %d (row %d) out of range", tokens[r], r);
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(m->device));
  int rc;
  if (rows == 1) {
    // no draft: the ordinary S=1 step of that sequence (the decode engine or the chain, same bits), so a call without drafts
    // costs exactly a plain step
    const int saved = s->active_seq;
    s->active_seq = seq[0];
    int32_t nxt = -1;
    rc = forward_locked(s, tokens, 1, start_pos[0], logits != nullptr, false, logits, &nxt);
    s->active_seq = saved;
    if (rc) return rc;
    if (next_out) next_out[0] = nxt;
    if (n_accepted) n_accepted[0] = 0;
    return 0;
  }
  const bool eng = spec_engine_ok(s, rows);
  if (!eng && !s->sdpa_smem_decode && !s->ss.sc)
    return fail(LNB_EINVAL, "speculative calls beyond the shared-memory attention kernel need head_dim <= 128 and n_rep <= 8");
  int32_t row_seq[8], row_pos[8];
  bool samp = false, lp = false, pen = false;
  for (int i = 0, r = 0; i < n_segs; i++)
    for (int k = 0; k <= n_draft[i]; k++, r++) {
      row_seq[r] = seq[i];
      row_pos[r] = start_pos[i] + k;
      samp |= processed(s, seq[i]);
      pen |= s->pen_on[seq[i]];
      lp |= s->lp_top[seq[i]] >= 0;
    }
  if (!s->d_rag) {   // the row map (shared with ragged calls)
    const cudaError_t e = cudaMalloc((void**)&s->d_rag, row_map_words(s->max_rows) * 4);
    if (e != cudaSuccess) {
      s->d_rag = nullptr;
      cudaGetLastError();
      return fail(LNB_ENOMEM, "speculative row map: %zu bytes of device memory asked for: %s", row_map_words(s->max_rows) * 4,
                  cudaGetErrorString(e));
    }
  }
  if (samp && (rc = samp_grow(s, rows))) return rc;
  if ((rc = ensure_logits(s, (size_t)rows))) return rc;
  s->kept_rows = 0;   // a logits handle is valid until the session's next forward
  // [tokens | row_seq | row_pos]: one pinned staging copy
  int32_t* h = s->h_tok;
  memcpy(h, tokens, (size_t)rows * 4);
  memcpy(h + rows, row_seq, (size_t)rows * 4);
  memcpy(h + 2 * rows, row_pos, (size_t)rows * 4);
  CU(cudaMemcpyAsync(s->d_rag, h, (size_t)3 * rows * 4, cudaMemcpyHostToDevice, s->stream));
  if (eng) {
    // ONE launch of the batch engine: every weight matrix streamed once for all rows
    if ((rc = launch_record(s, rows_spec(s, rows, pen)))) return rc;
    if ((rc = batch_engine_build(s, (logits || samp || lp) ? s->logits : nullptr))) return rc;
    if ((rc = batch_engine_launch(s, rows, s->d_rag, s->d_rag + 2 * rows, s->d_rag + rows))) return rc;
  } else {
    if ((rc = set_state(s, 0, rows, -1, false))) return rc;
    if ((rc = enqueue_forward(s, rows_spec(s, rows, pen)))) return rc;
  }
  int32_t p_next[8];
  for (int r = 0; r < rows; r++) p_next[r] = row_pos[r] + 1;
  if ((rc = call_tail(s, rows, 0, row_seq, p_next, s->d_next_arr, s->d_next_arr, logits, rows, s->d_next_arr))) return rc;
  // acceptance: row j of a segment predicts the token at position start + j + 1, which draft j + 1 claims
  for (int i = 0, r0 = 0; i < n_segs; r0 += 1 + n_draft[i], i++) {
    int acc = 0;
    while (acc < n_draft[i] && s->h_out[r0 + acc] == tokens[r0 + acc + 1]) acc++;
    if (n_accepted) n_accepted[i] = acc;
  }
  if (next_out) memcpy(next_out, s->h_out, (size_t)rows * 4);
  return 0;
}

extern "C" int lnb_decode_run(lnb_session* s, int32_t first_token, int start_pos, int n_steps, int use_graph,
                              int32_t* tokens_out, float* ms_out) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  if (n_steps <= 0 || start_pos < 0 || start_pos + n_steps > s->seq_len)
    return fail(LNB_EINVAL, "positions [%d, %d) exceed SequenceLength %d", start_pos, start_pos + n_steps, s->seq_len);
  if (first_token < 0 || first_token >= s->m->a.vocab_size) return fail(LNB_EINVAL, "token id %d out of range", first_token);
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(s->m->device));
  s->kept_rows = 0;   // a logits handle is valid until the session's next forward
  int rc;
  // a sampled sequence decodes on the kernel chain (the persistent engine feeds back the greedy token inside the kernel):
  // each step keeps its logits row and ends in the sampler, whose token is the next step's input.  A sequence with
  // logprobs on decodes on the chain too, each step then ending in the logprob job keyed on st->pos (= p_next).  A
  // penalized sequence records its token, runs the penalty job and draws from the sampler (greedy: its rank 0) each step.
  const int seq = s->active_seq;
  const bool pen = s->pen_on[seq], samp = processed(s, seq), greedy_slot = samp && !s->samp_on[seq];
  const bool lp = s->lp_top[seq] >= 0, keep = samp || lp;
  if (s->samp_on[seq] && engine_ok(s)) g_err = "the active sequence samples: lnb_decode_run runs the kernel chain (the decode engine has no sampler)";
  else if (pen && engine_ok(s))
    g_err = "the active sequence is penalized: lnb_decode_run runs the kernel chain (the decode engine keeps no token history)";
  else if (lp && engine_ok(s))
    g_err = "the active sequence has logprobs on: lnb_decode_run runs the kernel chain (the decode engine keeps no logits row)";
  if (!keep && engine_ok(s)) {
    // the whole run is ONE launch of the persistent engine: n_steps forwards, the greedy token fed back on the device
    if ((rc = engine_build(s, -1, nullptr))) return rc;
    if ((rc = set_state(s, start_pos, 1, first_token, true))) return rc;
    *s->h_err = 0;
    CU(cudaEventRecord(s->ev0, s->stream));
    if ((rc = engine_launch(s, n_steps, true))) return rc;
    CU(cudaEventRecord(s->ev1, s->stream));
    CU(cudaMemcpyAsync(s->h_out, s->d_tok_out, (size_t)n_steps * 4, cudaMemcpyDeviceToHost, s->stream));
    if ((rc = sync_stream(s))) return rc;
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
    if (ms_out) *ms_out = ms;
    if (tokens_out) memcpy(tokens_out, s->h_out, (size_t)n_steps * 4);
    return use_graph ? 1 : 0;   // (no graph is needed: there is nothing left to replay)
  }
  if (keep && (rc = ensure_logits(s, 1))) return rc;
  if (s->graph_tried && (s->graph_sampled != samp || s->graph_lp != lp || s->graph_pen != pen || s->graph_greedy != greedy_slot ||
                         (keep && s->graph_logits != s->logits)))
    drop_graph(s);
  if (lp) {   // the job's one row, read by every step (and by the graph's replays): the token st->next_token, record st->pos
    lp_row(s, 0, 0, &s->st->next_token, seq, 0, &s->st->pos);
    if ((rc = lp_upload(s, 1))) return rc;
  }
  auto step = [&]() -> int {
    int r = enqueue_forward(s, rows_single(s, 1, nullptr, keep ? 1 : 0, true, true));
    if (r) return r;
    const int32_t row = 0, pn = -1;
    if (samp && (r = launch_sample(s, 1, &row, &seq, &pn, nullptr, nullptr, true))) return r;
    return lp ? launch_logprob(s, 1) : 0;
  };
  if (use_graph && !s->graph && !s->graph_tried) {
    s->graph_tried = true;
    s->graph_sampled = samp;
    s->graph_lp = lp;
    s->graph_pen = pen;
    s->graph_greedy = greedy_slot;
    s->graph_logits = s->logits;
    cudaGraph_t g = nullptr;
    const int64_t saved = s->launches;
    cudaError_t e = cudaStreamBeginCapture(s->stream, cudaStreamCaptureModeThreadLocal);
    rc = 0;
    if (e == cudaSuccess) {
      rc = step();
      e = cudaStreamEndCapture(s->stream, &g);
    }
    if (e == cudaSuccess && rc == 0 && g) {
      e = cudaGraphInstantiate(&s->graph, g, 0);
      if (e != cudaSuccess) s->graph = nullptr;
    }
    if (g) cudaGraphDestroy(g);
    cudaGetLastError();
    s->graph_launches = s->launches - saved;   // the capture launched nothing: count it per replay
    s->launches = saved;
  }
  const bool graph = use_graph && s->graph;
  if ((rc = set_state(s, start_pos, 1, first_token, true))) return rc;
  CU(cudaEventRecord(s->ev0, s->stream));
  for (int i = 0; i < n_steps; i++) {
    if (graph) {
      CU(cudaGraphLaunch(s->graph, s->stream));
      s->launches += s->graph_launches;
    } else if ((rc = step())) {
      return rc;
    }
  }
  CU(cudaEventRecord(s->ev1, s->stream));
  CU(cudaMemcpyAsync(s->h_out, s->d_tok_out, (size_t)n_steps * 4, cudaMemcpyDeviceToHost, s->stream));
  if ((rc = p2p_err_enqueue(s))) return rc;
  CU(cudaStreamSynchronize(s->stream));
  CU(cudaGetLastError());
  if ((rc = p2p_err_check(s))) return rc;
  float ms = 0.f;
  CU(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
  if (ms_out) *ms_out = ms;
  if (tokens_out) memcpy(tokens_out, s->h_out, (size_t)n_steps * 4);
  return graph ? 1 : 0;
}

// Times one projection kernel of the decode step in isolation: launches it for every layer's
// weights back to back (n_layers * 100+ MB >> L2, so every launch streams from HBM), `reps`
// sweeps, CUDA events on the session stream.  kind: 0 = wq|wk|wv, 1 = wo, 2 = w1|w3, 3 = w2,
// 4 = LM head.  Outputs go to the session's scratch activations (results are discarded).
extern "C" int lnb_session_bench_kernel(lnb_session* s, int kind, int reps, float* ms_per_launch, int64_t* bytes_per_launch,
                                        int* launches) {
  if (!s || reps <= 0 || kind < 0 || kind > 4) return fail(LNB_EINVAL, "bad argument");
  std::lock_guard<std::mutex> lk(s->mu);
  lnb_model* m = s->m;
  const lnb_model_args& a = m->a;
  CU(cudaSetDevice(m->device));
  if (engine_ok(s)) {
    // the projection as the decode step runs it: a phase of the persistent engine (balanced static row split, weights
    // prefetched across the grid barrier).  One launch walks all layers' copies `reps` times; time per phase.
    int rc = engine_build(s, kind, nullptr);
    if (rc) return rc;
    if ((rc = set_state(s, 0, 1, 0, false))) return rc;
    *s->h_err = 0;
    if ((rc = engine_launch(s, 1, false))) return rc;     // warm-up sweep
    if ((rc = set_state(s, 0, 1, 0, false))) return rc;
    CU(cudaEventRecord(s->ev0, s->stream));
    if ((rc = engine_launch(s, reps, false))) return rc;
    CU(cudaEventRecord(s->ev1, s->stream));
    if ((rc = sync_stream(s))) return rc;
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
    const int n = s->n_phases * reps;
    int64_t bytes = 0;
    switch (kind) {
      case 0: bytes = (int64_t)(m->q_l + 2 * m->kv_l) * a.dim * 2; break;
      case 1: bytes = (int64_t)a.dim * m->q_l * 2; break;
      case 2: bytes = (int64_t)2 * m->ffn_l * a.dim * 2; break;
      case 3: bytes = (int64_t)a.dim * m->ffn_l * 2; break;
      default: bytes = (int64_t)m->vocab_l * a.dim * 2; break;
    }
    // packed phases read what their units hold: the mean over the phases of the sweep
    std::vector<EnginePhase> hp(s->n_phases);
    CU(cudaMemcpy(hp.data(), s->d_phases, hp.size() * sizeof(EnginePhase), cudaMemcpyDeviceToHost));
    if (!hp.empty() && hp[0].Wp) {
      int64_t sum = 0;
      for (int i = 0; i < s->n_phases; i++) {
        const lnb_model::WPack& wp = (kind == 4) ? m->wp_out : m->wp_w13[i];
        sum += hp[i].Wp ? wp.read_bytes : bytes;
      }
      bytes = sum / s->n_phases;
    }
    if (ms_per_launch) *ms_per_launch = ms / (float)n;
    if (bytes_per_launch) *bytes_per_launch = bytes;
    if (launches) *launches = n;
    s->eng_key_kind = -2;   // the next decode call rebuilds the step's phase list
    return 0;
  }
  const Launcher L{s->stream, LAUNCH_PDL, &s->launches};
  if (int rc0 = set_state(s, 0, 1, 0, false)) return rc0;
  int n_launch = 0;
  int64_t bytes = 0;
  auto sweep = [&]() -> int {
    int rc = 0;
    const int nl = (kind == 4) ? 4 : a.n_layers;  // the LM head is one 1 GB matrix: repeat it
    for (int l = 0; l < nl && !rc; l++) {
      LayerW& W = m->layers[kind == 4 ? 0 : l];
      GemvParams p{};
      p.eps = a.norm_eps;
      p.rscale = (s->mode == LNB_ACC_STRICT) ? s->rs : nullptr;
      switch (kind) {
        case 0:
          p.W = W.wqkv; p.N = m->q_l + 2 * m->kv_l; p.K = a.dim; p.x = s->x; p.ldx = a.dim; p.norm_w = W.attn_norm;
          p.out_bf16 = s->q; p.ldo = m->q_l; p.q_dim = m->q_l; p.kv_dim = m->kv_l; p.head_dim = a.head_dim;
          p.cache_k = s->ck[l]; p.cache_v = s->cv[l]; p.cis = m->cis; p.pos_ptr = &s->st->pos;
          rc = launch_gemv<PRO_RMSNORM, EPI_QKV_ROPE>(L, s->mode, p, 1);
          break;
        case 1:
          p.W = W.wo; p.N = a.dim; p.K = m->q_l; p.x = s->o; p.ldx = m->q_l; p.ldo = a.dim; p.out_bf16 = s->h1; p.res = s->x;
          rc = launch_gemv<PRO_PLAIN, EPI_RESID>(L, s->mode, p, 1);
          break;
        case 2:
          p.W = W.w13; p.N = 2 * m->ffn_l; p.K = a.dim; p.x = s->h1; p.ldx = a.dim; p.norm_w = W.ffn_norm;
          p.out_bf16 = s->mbuf; p.ldo = m->ffn_l; p.silu_tab = m->silu_tab;
          rc = launch_gemv<PRO_RMSNORM, EPI_SWIGLU>(L, s->mode, p, 1);
          break;
        case 3:
          p.W = W.w2; p.N = a.dim; p.K = m->ffn_l; p.x = s->mbuf; p.ldx = m->ffn_l; p.ldo = a.dim; p.out_bf16 = s->h1; p.res = s->x;
          rc = launch_gemv<PRO_PLAIN, EPI_RESID>(L, s->mode, p, 1);
          break;
        case 4:
          p.W = m->output; p.N = m->vocab_l; p.K = a.dim; p.x = s->x; p.ldx = a.dim; p.norm_w = m->norm; p.ldo = m->vocab_l;
          p.st = nullptr; p.argmax_row = -1;
          rc = launch_gemv<PRO_RMSNORM, EPI_LOGITS>(L, s->mode, p, 1);
          break;
      }
      bytes = (int64_t)p.N * p.K * 2;
      n_launch++;
    }
    return rc;
  };
  if (s->mode == LNB_ACC_STRICT) {
    int rc0 = launch_rms_scale(L, (const uint16_t*)s->x, a.dim, s->rs, 1, a.dim, a.norm_eps);
    if (rc0) return rc0;
  }
  int rc = sweep();  // warm-up sweep
  if (rc) return rc;
  n_launch = 0;
  CU(cudaEventRecord(s->ev0, s->stream));
  for (int r = 0; r < reps; r++)
    if ((rc = sweep())) return rc;
  CU(cudaEventRecord(s->ev1, s->stream));
  CU(cudaStreamSynchronize(s->stream));
  CU(cudaGetLastError());
  float ms = 0.f;
  CU(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
  if (ms_per_launch) *ms_per_launch = ms / (float)n_launch;
  if (bytes_per_launch) *bytes_per_launch = bytes;
  if (launches) *launches = n_launch;
  return 0;
}

// LNB_ENGINE_PROF=1: cycle sums of the engine's consumer thread 0, averaged and maximised over the CTAs, since the last
// call; out[2 * 8] = {mean, max} x {grid barrier, prologue, main loop, combine + epilogue, attention, peer reduce, -, -}
// 1: this session's S=1 steps run as the persistent decode engine; 0: as the kernel chain (lnb_last_error says why)
extern "C" int lnb_session_decode_engine(lnb_session* s) {
  if (!s) return fail(LNB_EINVAL, "session is NULL");
  std::lock_guard<std::mutex> lk(s->mu);
  CU(cudaSetDevice(s->m->device));
  if (engine_ok(s)) return 1;
  g_err = s->eng_state < 0 ? s->eng_why : !s->eng_single_default ? std::string("single-GPU FAST: the kernel chain is the default") : std::string("tensor-parallel session without the peer all-reduce (NCCL collectives cannot run inside a kernel)");
  return 0;
}
extern "C" int lnb_session_engine_profile(lnb_session* s, double* out16) {   // (out: 2 * ENG_NPROF doubles)
  if (!s || !out16) return fail(LNB_EINVAL, "NULL argument");
  if (!s->d_prof) return fail(LNB_ESTATE, "no engine profile (set LNB_ENGINE_PROF=1 before the session's first decode)");
  CU(cudaSetDevice(s->m->device));
  CU(cudaStreamSynchronize(s->stream));
  const int G = s->m->sm_count;
  std::vector<unsigned long long> h((size_t)G * ENG_NPROF);
  CU(cudaMemcpy(h.data(), s->d_prof, h.size() * 8, cudaMemcpyDeviceToHost));
  CU(cudaMemset(s->d_prof, 0, h.size() * 8));
  for (int k = 0; k < ENG_NPROF; k++) {
    double sum = 0, mx = 0;
    for (int b = 0; b < G; b++) {
      const double v = (double)h[(size_t)b * ENG_NPROF + k];
      sum += v;
      mx = std::max(mx, v);
    }
    out16[2 * k] = sum / G;
    out16[2 * k + 1] = mx;
  }
  return 0;
}

extern "C" int lnb_session_read(lnb_session* s, int which, int layer, void* host, int64_t nbytes) {
  if (!s || !host) return fail(LNB_EINVAL, "NULL argument");
  lnb_model* m = s->m;
  CU(cudaSetDevice(m->device));
  const void* src = nullptr;
  int64_t avail = 0;
  switch (which) {
    case LNB_BUF_RESIDUAL:
      if (s->last_was_engine) {   // the engine keeps the residual stream as tagged words: strip the tags
        if (nbytes > (int64_t)m->a.dim * 2) return fail(LNB_EINVAL, "the decode engine keeps one row");
        std::vector<uint32_t> t((size_t)m->a.dim);
        CU(cudaStreamSynchronize(s->stream));
        CU(cudaMemcpy(t.data(), s->x_t, t.size() * 4, cudaMemcpyDeviceToHost));
        uint16_t* o = (uint16_t*)host;
        for (int64_t i = 0; i < nbytes / 2; i++) o[i] = (uint16_t)(t[(size_t)i] & 0xffffu);
        return 0;
      }
      src = s->x; avail = (int64_t)s->max_rows * m->a.dim * 2; break;
    case LNB_BUF_CACHE_K:
    case LNB_BUF_CACHE_V:
      if (layer < 0 || layer >= m->a.n_layers) return fail(LNB_EINVAL, "bad layer %d", layer);
      src = (which == LNB_BUF_CACHE_K ? s->ck[layer] : s->cv[layer]) + (size_t)s->active_seq * s->seq_len * m->kv_l;
      avail = (int64_t)s->seq_len * m->kv_l * 2;
      break;
    case LNB_BUF_LOGITS: src = s->logits; avail = (int64_t)s->logits_rows * m->vocab_l * 4; break;
    default: return fail(LNB_EINVAL, "bad buffer id %d", which);
  }
  if (!src || nbytes > avail) return fail(LNB_EINVAL, "buffer %d holds %lld bytes, %lld requested", which, (long long)avail, (long long)nbytes);
  CU(cudaStreamSynchronize(s->stream));
  CU(cudaMemcpy(host, src, (size_t)nbytes, cudaMemcpyDeviceToHost));
  return 0;
}

// ------------------------------------------------------------------------------------------
// op-level API: host pointers in / out, staged through HBM, same kernels as the model path
// Device scratch for the op-level calls: a grow-only per-thread arena (cudaMalloc / cudaFree per
// call cost more than the kernels they serve).  Buffers are carved with 256-byte alignment and
// the arena is rewound at the start of every op.
struct OpArena {
  uint8_t* base = nullptr;
  size_t cap = 0, used = 0;
  int dev = -1;
  std::vector<void*> overflow;  // blocks allocated after the arena filled up in this op
  void rewind() {
    for (void* q : overflow) cudaFree(q);
    overflow.clear();
    used = 0;
  }
  void* take(size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    int d = 0;
    cudaGetDevice(&d);
    if (d != dev) {  // the calling thread switched devices: start over
      if (base) cudaFree(base);
      base = nullptr; cap = used = 0; dev = d;
    }
    if (used + bytes > cap) {
      if (used == 0) {  // nothing handed out yet: regrow the arena itself
        if (base) cudaFree(base);
        base = nullptr;
        const size_t want = bytes * 2 > ((size_t)8 << 20) ? bytes * 2 : ((size_t)8 << 20);
        if (cudaMalloc((void**)&base, want) != cudaSuccess) { cap = 0; return nullptr; }
        cap = want;
      } else {
        void* q = nullptr;
        if (cudaMalloc(&q, bytes) != cudaSuccess) return nullptr;
        overflow.push_back(q);
        return q;
      }
    }
    void* r = base + used;
    used += bytes;
    return r;
  }
};
static thread_local OpArena g_arena;
struct DevBuf {
  void* p = nullptr;
  cudaError_t alloc(size_t bytes) {
    p = g_arena.take(bytes ? bytes : 16);
    return p ? cudaSuccess : cudaErrorMemoryAllocation;
  }
  template <class T> T* as() { return reinterpret_cast<T*>(p); }
};
struct OpScope {  // rewinds the arena when an op-level entry point begins
  OpScope() { g_arena.rewind(); }
};
#define OPBUF(buf, bytes)                                                                     \
  DevBuf buf;                                                                                 \
  { cudaError_t e_ = buf.alloc(bytes); if (e_ != cudaSuccess) return fail(LNB_ENOMEM, "cudaMalloc(%zu): %s", (size_t)(bytes), cudaGetErrorString(e_)); }
#define H2D(buf, host, bytes) CU(cudaMemcpy(buf.p, host, bytes, cudaMemcpyHostToDevice))
#define D2H(host, buf, bytes) CU(cudaMemcpy(host, buf.p, bytes, cudaMemcpyDeviceToHost))
static int op_finish() {
  CU(cudaGetLastError());
  CU(cudaDeviceSynchronize());
  return 0;
}
static int grid_for(int64_t n) { return (int)std::min<int64_t>(kWaveSMs * 8, (n + 255) / 256); }

extern "C" int lnb_op_linear_bf16(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int K, int N, int acc_mode) {
  OpScope scope_;
  if (!x || !w || !out) return fail(LNB_EINVAL, "NULL argument");
  if (S <= 0 || K <= 0 || N <= 0) return fail(LNB_EINVAL, "non-positive shape");
  if (acc_mode != LNB_ACC_STRICT && acc_mode != LNB_ACC_FAST) return fail(LNB_EINVAL, "bad acc_mode %d", acc_mode);
  const size_t xb = (size_t)S * K * 2, wb = (size_t)N * K * 2, ob = (size_t)S * N * 2;
  OPBUF(dx, xb); OPBUF(dw, wb); OPBUF(dout, ob);
  H2D(dx, x, xb); H2D(dw, w, wb);
  const bool tileable = (N % 16 == 0) && (K % 8 == 0) && (CfgF1::smem_bytes(K) <= kMaxSmem);
  if (acc_mode == LNB_ACC_FAST && tc_eligible(S, N, K)) {
    // prompt-sized inputs: wgmma tensor-core tiles (hardware accumulation order)
    const int Mpad = (S + TC_BM - 1) / TC_BM * TC_BM;
    OPBUF(dwp, wb); OPBUF(dx8, (size_t)Mpad * K * 2);
    retile_kernel<<<grid_for((int64_t)N * K / 8), 256>>>(dw.as<uint16_t>(), K, 0, 0, N, K, dwp.as<uint16_t>(), 0, 1);
    pack_x8_kernel<<<grid_for((int64_t)Mpad * K / 8), 256>>>(dx.as<uint16_t>(), K, S, Mpad, K, dx8.as<uint16_t>());
    GemmTcParams g{};
    g.X8 = dx8.as<uint16_t>(); g.W = dwp.as<uint16_t>(); g.M = S; g.N = N; g.K = K; g.out_bf16 = dout.as<uint16_t>(); g.ldo = N;
    Launcher L{nullptr, LAUNCH_PLAIN, nullptr};
    int rc = launch_gemm_tc<TC_EPI_BF16>(L, g);
    if (rc) return rc;
    rc = op_finish();
    if (rc) return rc;
    D2H(out, dout, ob);
    return 0;
  }
  if (!tileable) {
    // shapes outside the panel layout (e.g. the reference's 2x3 . 4x3^T test): reference order, one thread per output
    linear_naive_kernel<<<(int)(((int64_t)S * N + 255) / 256), 256>>>(dx.as<uint16_t>(), dw.as<uint16_t>(), dout.as<uint16_t>(), S, K, N);
  } else {
    OPBUF(dwp, wb);
    retile_kernel<<<grid_for((int64_t)N * K / 8), 256>>>(dw.as<uint16_t>(), K, 0, 0, N, K, dwp.as<uint16_t>(), 0, 1);
    GemvParams p{};
    p.W = dwp.as<uint16_t>(); p.N = N; p.K = K; p.x = dx.as<uint16_t>(); p.ldx = K; p.out_bf16 = dout.as<uint16_t>(); p.ldo = N;
    Launcher L{nullptr, LAUNCH_PLAIN, nullptr};
    int rc = launch_gemv<PRO_PLAIN, EPI_BF16>(L, acc_mode, p, S);
    if (rc) return rc;
    rc = op_finish();
    if (rc) return rc;
    D2H(out, dout, ob);
    return 0;
  }
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, ob);
  return 0;
}

extern "C" int lnb_op_matmul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int B, int M, int K, int N) {
  OpScope scope_;
  if (!a || !b || !out) return fail(LNB_EINVAL, "NULL argument");
  if (B <= 0 || M <= 0 || K <= 0 || N <= 0) return fail(LNB_EINVAL, "non-positive shape");
  const size_t ab = (size_t)B * M * K * 2, bb = (size_t)B * K * N * 2, ob = (size_t)B * M * N * 2;
  OPBUF(da, ab); OPBUF(db, bb); OPBUF(dout, ob);
  H2D(da, a, ab); H2D(db, b, bb);
  matmul_naive_kernel<<<(int)(((int64_t)B * M * N + 255) / 256), 256>>>(da.as<uint16_t>(), db.as<uint16_t>(), dout.as<uint16_t>(), B, M, K, N);
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, ob);
  return 0;
}

extern "C" int lnb_op_rmsnorm_bf16(const uint16_t* x, const uint16_t* w, uint16_t* out, int S, int D, float eps, int acc_mode) {
  OpScope scope_;
  if (!x || !w || !out) return fail(LNB_EINVAL, "NULL argument");
  if (S <= 0 || D <= 0) return fail(LNB_EINVAL, "non-positive shape");
  const size_t xb = (size_t)S * D * 2;
  OPBUF(dx, xb); OPBUF(dw, (size_t)D * 2); OPBUF(dout, xb);
  H2D(dx, x, xb); H2D(dw, w, (size_t)D * 2);
  const bool strict = (acc_mode == LNB_ACC_STRICT);
  const float* rs = nullptr;
  OPBUF(drs, (size_t)S * 4);
  if (strict && D % 2 == 0 && (size_t)D * 4 <= 48 * 1024) {  // the model path's own scale kernel
    const Launcher L{nullptr, LAUNCH_PLAIN, nullptr};
    int rc0 = launch_rms_scale(L, dx.as<uint16_t>(), D, drs.as<float>(), S, D, eps);
    if (rc0) return rc0;
    rs = drs.as<float>();
  }
  rmsnorm_kernel<<<S, 256>>>(dx.as<uint16_t>(), dw.as<uint16_t>(), dout.as<uint16_t>(), D, eps, strict ? 1 : 0, rs);
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, xb);
  return 0;
}

extern "C" int lnb_op_rms_scale_f32(const uint16_t* x, float* r, int S, int D, float eps, int algo) {
  OpScope scope_;
  if (!x || !r) return fail(LNB_EINVAL, "NULL argument");
  if (S <= 0 || D <= 0 || (D & 1)) return fail(LNB_EINVAL, "bad shape");
  if (algo < RMS_AUTO || algo > RMS_ENGINE) return fail(LNB_EINVAL, "bad algo %d", algo);
  if (algo == RMS_ENGINE) {
    int ech = 0, ent = 0;
    if (!eng_scan_shape(D, &ech, &ent) || (size_t)D * 4 + 4096 > 200 * 1024) return fail(LNB_EINVAL, "row length %d does not fit the engine's scan", D);
    const size_t xb2 = (size_t)S * D * 2;
    OPBUF(dx2, xb2); OPBUF(dr2, (size_t)S * 4);
    H2D(dx2, x, xb2);
    const size_t smem = (size_t)D * 4 + 4096;
    const auto kern = ech == 16 ? eng_rms_scale_kernel<16>
                    : ech == 8  ? eng_rms_scale_kernel<8>
                    : ech == 4  ? eng_rms_scale_kernel<4>
                                : eng_rms_scale_kernel<2>;
    CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const Launcher L{nullptr, LAUNCH_PLAIN, nullptr};
    int rc2 = launch_kernel(L, kern, dim3(S), dim3(ENG_NCONS), smem, (const uint16_t*)dx2.as<uint16_t>(), D, dr2.as<float>(), D, eps);
    if (rc2) return rc2;
    rc2 = op_finish();
    if (rc2) return rc2;
    D2H(r, dr2, (size_t)S * 4);
    return 0;
  }
  int ch, nt;
  const bool fits = seq_scan_shape(D, &ch, &nt);
  if ((algo == RMS_SCAN || algo == RMS_SEG) && !fits) return fail(LNB_EINVAL, "row length %d does not fit the scan kernels", D);
  if ((size_t)D * 4 > 48 * 1024 && (algo == RMS_CHAIN || !fits)) return fail(LNB_EINVAL, "row length %d too long", D);
  const size_t xb = (size_t)S * D * 2;
  OPBUF(dx, xb); OPBUF(dr, (size_t)S * 4);
  H2D(dx, x, xb);
  const Launcher L{nullptr, LAUNCH_PLAIN, nullptr};
  int rc = launch_rms_scale(L, dx.as<uint16_t>(), D, dr.as<float>(), S, D, eps, algo);
  if (rc) return rc;
  rc = op_finish();
  if (rc) return rc;
  D2H(r, dr, (size_t)S * 4);
  return 0;
}

extern "C" int lnb_op_rope_bf16(const uint16_t* x, const float* cis, uint16_t* out, int S, int H, int hd, int start_pos) {
  OpScope scope_;
  if (!x || !cis || !out) return fail(LNB_EINVAL, "NULL argument");
  if (S <= 0 || H <= 0 || hd <= 0 || (hd & 1) || start_pos < 0) return fail(LNB_EINVAL, "bad shape");
  const size_t xb = (size_t)S * H * hd * 2, cb = (size_t)(start_pos + S) * (hd / 2) * 2 * 4;
  OPBUF(dx, xb); OPBUF(dc, cb); OPBUF(dout, xb);
  H2D(dx, x, xb); H2D(dc, cis, cb);
  rope_kernel<<<grid_for((int64_t)S * H * hd / 2), 256>>>(dx.as<uint16_t>(), dc.as<float>(), dout.as<uint16_t>(), S, H, hd, start_pos);
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, xb);
  return 0;
}

extern "C" int lnb_op_attention_bf16(const uint16_t* q, const uint16_t* cache_k, const uint16_t* cache_v, uint16_t* out,
                                     int S, int T, int n_heads, int n_kv, int hd, int causal_mask, int acc_mode) {
  OpScope scope_;
  if (!q || !cache_k || !cache_v || !out) return fail(LNB_EINVAL, "NULL argument");
  if (S <= 0 || T < S || n_heads <= 0 || n_kv <= 0 || n_heads % n_kv || hd <= 0 || hd % 8) return fail(LNB_EINVAL, "bad shape");
  if (causal_mask < 0 || causal_mask > 2) return fail(LNB_EINVAL, "bad causal_mask %d", causal_mask);
  if (causal_mask == 1 && T != S) return fail(LNB_EINVAL, "causal mask needs T == S (reference mask is [S,S])");
  const size_t smem = (size_t)T * 12 + (size_t)hd * 4;
  // beyond sdpa_kernel's T limit the op routes as a long session does: FAST prompts of >= 32 rows keep the tiled prompt
  // kernels (they stream key tiles), every other case runs the streamed kernel
  const bool fits = smem <= 200 * 1024;
  const bool tiled = acc_mode == LNB_ACC_FAST && S > 1 && causal_mask && hd == SP_HD && (n_heads * hd) % 128 == 0 && (fits || S >= 32);
  if (!fits && !tiled && !ss_shape_ok(hd, n_heads / n_kv)) return fail(LNB_EINVAL, "T %d too long", T);
  const size_t qb = (size_t)S * n_heads * hd * 2, cb = (size_t)T * n_kv * hd * 2;
  OPBUF(dq, qb); OPBUF(dk, cb); OPBUF(dv, cb); OPBUF(dout, qb);
  H2D(dq, q, qb); H2D(dk, cache_k, cb); H2D(dv, cache_v, cb);
  CU(cudaFuncSetAttribute(sdpa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  const float f = attn_scale_bf16(hd);
  if (!fits && !tiled) {
    SsScratch x;
    size_t sc_b, z_b, op_b;
    ss_plan(x, T, S, n_heads, hd, &sc_b, &z_b, &op_b);
    OPBUF(dsc, sc_b); OPBUF(dz, z_b); OPBUF(dop, op_b);
    x.sc = dsc.as<uint16_t>(); x.z = dz.as<double>(); x.op = dop.as<float>();
    StreamAttn P{};
    P.q = dq.as<uint16_t>(); P.ldq = n_heads * hd;
    P.cache_k = dk.as<uint16_t>(); P.cache_v = dv.as<uint16_t>(); P.kv_dim = n_kv * hd;
    P.n_rep = n_heads / n_kv; P.hd = hd; P.n_heads = n_heads;
    P.pos_fixed = causal_mask ? T - S : T - 1; P.pos_step = causal_mask ? 1 : 0;   // query row s at T - S + s
    P.out = dout.as<uint16_t>(); P.ldo = n_heads * hd;
    P.scale = f;
    P.strict = acc_mode == LNB_ACC_STRICT ? 1 : 0;
    int rc2 = launch_stream_attn(Launcher{nullptr, LAUNCH_PLAIN, nullptr}, P, S, n_kv, x);
    if (!rc2) rc2 = op_finish();
    if (rc2) return rc2;
    D2H(out, dout, qb);
    return 0;
  }
  if (tiled) {
    // the prefill path's tiled two-pass kernel (writes the X8 operand of the Wo GEMM; unpacked here); query row s sits at
    // position (T - S) + s, as in a session's chunked prefill
    const int Mpad = (S + 127) / 128 * 128;
    const int32_t pos0 = T - S;
    OPBUF(d8, (size_t)Mpad * n_heads * hd * 2); OPBUF(dpos, 16);
    H2D(dpos, &pos0, sizeof(pos0));
    const double* exp_tab = (sdpa_tc_enabled() && S >= 32) ? exp_table_device() : nullptr;
    if (exp_tab) {
      CU(cudaFuncSetAttribute(sdpa_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ST_SMEM));
      sdpa_tc_kernel<<<dim3(n_heads, (S + 127) / 128), 256, ST_SMEM>>>(dq.as<uint16_t>(), n_heads * hd, dk.as<uint16_t>(), dv.as<uint16_t>(),
                                                                       n_kv * hd, n_heads / n_kv, d8.as<uint16_t>(), n_heads * hd,
                                                                       dpos.as<int32_t>(), S, f, exp_tab);
    } else {
      CU(cudaFuncSetAttribute(sdpa_prefill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SP_SMEM));
      sdpa_prefill_kernel<<<dim3(n_heads, (S + SP_QB - 1) / SP_QB), 256, SP_SMEM>>>(dq.as<uint16_t>(), n_heads * hd, dk.as<uint16_t>(),
                                                                                    dv.as<uint16_t>(), n_kv * hd, n_heads / n_kv,
                                                                                    d8.as<uint16_t>(), n_heads * hd, dpos.as<int32_t>(), S, f);
    }
    unpack_x8_kernel<<<grid_for((int64_t)S * n_heads * hd / 8), 256>>>(d8.as<uint16_t>(), S, n_heads * hd, dout.as<uint16_t>(), n_heads * hd);
    int rc2 = op_finish();
    if (rc2) return rc2;
    D2H(out, dout, qb);
    return 0;
  }
  sdpa_kernel<<<dim3(n_heads, S), 128, smem>>>(dq.as<uint16_t>(), n_heads * hd, dk.as<uint16_t>(), dv.as<uint16_t>(), n_kv * hd,
                                                n_heads / n_kv, hd, dout.as<uint16_t>(), n_heads * hd, nullptr, T - S, S,
                                                causal_mask ? 1 : 0, acc_mode == LNB_ACC_STRICT ? 1 : 0, f, 0);
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, qb);
  return 0;
}

static int silu_table_device(uint16_t** out) {
  static uint16_t* tab = nullptr;  // per process, device 0 of the calling thread's current device
  static int tab_dev = -1;
  int dev = 0;
  CU(cudaGetDevice(&dev));
  if (!tab || tab_dev != dev) {
    std::vector<uint16_t> h;
    build_silu_table(h);
    CU(cudaMalloc((void**)&tab, 65536 * 2));
    CU(cudaMemcpy(tab, h.data(), 65536 * 2, cudaMemcpyHostToDevice));
    tab_dev = dev;
  }
  *out = tab;
  return 0;
}

extern "C" int lnb_op_silu_bf16(const uint16_t* x, uint16_t* out, int64_t n) {
  OpScope scope_;
  if (!x || !out || n < 0) return fail(LNB_EINVAL, "bad argument");
  if (n == 0) return 0;
  uint16_t* tab;
  int rc = silu_table_device(&tab);
  if (rc) return rc;
  OPBUF(dx, (size_t)n * 2); OPBUF(dout, (size_t)n * 2);
  H2D(dx, x, (size_t)n * 2);
  silu_kernel<<<grid_for(n), 256>>>(dx.as<uint16_t>(), tab, dout.as<uint16_t>(), n);
  rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, (size_t)n * 2);
  return 0;
}

static int binary_op(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n, bool is_add) {
  OpScope scope_;
  if (!a || !b || !out || n < 0) return fail(LNB_EINVAL, "bad argument");
  if (n == 0) return 0;
  OPBUF(da, (size_t)n * 2); OPBUF(db, (size_t)n * 2); OPBUF(dout, (size_t)n * 2);
  H2D(da, a, (size_t)n * 2); H2D(db, b, (size_t)n * 2);
  if (is_add) add_kernel<<<grid_for(n), 256>>>(da.as<uint16_t>(), db.as<uint16_t>(), dout.as<uint16_t>(), n);
  else mul_kernel<<<grid_for(n), 256>>>(da.as<uint16_t>(), db.as<uint16_t>(), dout.as<uint16_t>(), n);
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, (size_t)n * 2);
  return 0;
}
extern "C" int lnb_op_add_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n) { return binary_op(a, b, out, n, true); }
extern "C" int lnb_op_mul_bf16(const uint16_t* a, const uint16_t* b, uint16_t* out, int64_t n) { return binary_op(a, b, out, n, false); }

extern "C" int lnb_op_softmax_f32(const float* x, float* out, int rows, int cols) {
  OpScope scope_;
  if (!x || !out || rows <= 0 || cols <= 0) return fail(LNB_EINVAL, "bad argument");
  const size_t b = (size_t)rows * cols * 4;
  OPBUF(dx, b); OPBUF(dout, b);
  H2D(dx, x, b);
  softmax_f32_kernel<<<rows, 256>>>(dx.as<float>(), dout.as<float>(), cols);
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, b);
  return 0;
}

extern "C" int lnb_op_argmax_f32(const float* x, int rows, int cols, int32_t* out) {
  OpScope scope_;
  if (!x || !out || rows <= 0 || cols <= 0) return fail(LNB_EINVAL, "bad argument");
  const size_t b = (size_t)rows * cols * 4;
  OPBUF(dx, b); OPBUF(dout, (size_t)rows * 4);
  H2D(dx, x, b);
  argmax_f32_kernel<<<rows, 256>>>(dx.as<float>(), cols, dout.as<int32_t>());
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, (size_t)rows * 4);
  return 0;
}

// the sampler alone on host rows: logits[rows, vocab], parameters p[rows], p_next pos_next[rows] -> out[rows]
extern "C" int lnb_op_sample_f32(const float* logits, int rows, int vocab, const lnb_sampling* p, const int32_t* pos_next, int32_t* out) {
  OpScope scope_;
  if (!logits || !p || !pos_next || !out) return fail(LNB_EINVAL, "NULL argument");
  if (rows < 1 || rows > SMP_MAX_ROWS || vocab < 1) return fail(LNB_EINVAL, "rows %d must be in [1, %d] and vocab %d positive", rows, SMP_MAX_ROWS, vocab);
  int rc;
  for (int r = 0; r < rows; r++) {
    if ((rc = sampling_check(p + r))) return rc;
    if (pos_next[r] < 0) return fail(LNB_EINVAL, "pos_next[%d] = %d must be >= 0", r, pos_next[r]);
  }
  const size_t b = (size_t)rows * vocab * 4;
  OPBUF(dx, b); OPBUF(dp, (size_t)rows * sizeof(lnb_sampling)); OPBUF(dw, (size_t)rows * vocab * 8); OPBUF(dout, (size_t)rows * 4);
  OPBUF(dc, (size_t)rows * (SMP_MERGE * 8 + 4));
  H2D(dx, logits, b);
  H2D(dp, p, (size_t)rows * sizeof(lnb_sampling));
  CU(cudaMemset(dc.p, 0, (size_t)rows * (SMP_MERGE * 8 + 4)));
  SampleJob J{};
  J.logits = dx.as<float>(); J.ld = vocab; J.V = vocab; J.n = rows;
  J.params = dp.as<lnb_sampling>(); J.wbuf = dw.as<unsigned long long>(); J.out = dout.as<int32_t>();
  J.cand = dc.as<unsigned long long>(); J.cnt = reinterpret_cast<unsigned int*>(J.cand + (size_t)rows * SMP_MERGE);
  for (int r = 0; r < rows; r++) { J.row[r] = r; J.slot[r] = r; J.p_next[r] = pos_next[r]; J.out_idx[r] = r; }
  if ((rc = launch_sample_job(Launcher{nullptr, LAUNCH_PLAIN, nullptr}, J))) return rc;
  if ((rc = op_finish())) return rc;
  D2H(out, dout, (size_t)rows * 4);
  return 0;
}

// the logprob kernels alone on host rows: logits[rows, vocab], targets[rows], one top_n -> out[rows]
extern "C" int lnb_op_logprobs_f32(const float* logits, int rows, int vocab, const int32_t* targets, int top_n, lnb_logprob* out) {
  OpScope scope_;
  if (!logits || !targets || !out) return fail(LNB_EINVAL, "NULL argument");
  if (rows < 1 || vocab < 1 || vocab > LP_MAX_VOCAB) return fail(LNB_EINVAL, "rows %d must be >= 1 and vocab %d in [1, %d]", rows, vocab, LP_MAX_VOCAB);
  if (top_n < 0 || top_n > LNB_LOGPROBS_TOP_MAX) return fail(LNB_EINVAL, "top_n %d must be in [0, %d]", top_n, LNB_LOGPROBS_TOP_MAX);
  for (int r = 0; r < rows; r++)
    if (targets[r] < 0 || targets[r] >= vocab) return fail(LNB_EINVAL, "targets[%d] = %d out of range", r, targets[r]);
  const int G = (vocab + LP_SLICE - 1) / LP_SLICE;
  const size_t b = (size_t)rows * vocab * 4, b_cand = (size_t)rows * G * (LP_TOP * 8 + 4) + (size_t)rows * 4;
  OPBUF(dx, b); OPBUF(dt, (size_t)rows * 4); OPBUF(dtop, 4); OPBUF(drows, (size_t)rows * sizeof(LpRow));
  OPBUF(drec, (size_t)rows * sizeof(LpRecord)); OPBUF(dc, b_cand);
  H2D(dx, logits, b);
  H2D(dt, targets, (size_t)rows * 4);
  H2D(dtop, &top_n, 4);
  CU(cudaMemset(dc.p, 0, b_cand));
  std::vector<LpRow> hr((size_t)rows);
  for (int r = 0; r < rows; r++)
    hr[r] = LpRow{dx.as<float>() + (size_t)r * vocab, dt.as<int32_t>() + r, drec.as<LpRecord>() + r, nullptr, 0, 0};
  H2D(drows, hr.data(), (size_t)rows * sizeof(LpRow));
  LogprobJob J{};
  J.rows = drows.as<LpRow>(); J.top_n = dtop.as<int32_t>(); J.V = vocab;
  J.cand = dc.as<unsigned long long>();
  J.above = reinterpret_cast<unsigned int*>(J.cand + (size_t)rows * G * LP_TOP);
  J.done = J.above + (size_t)rows * G;
  int rc;
  if ((rc = launch_logprob_job(Launcher{nullptr, LAUNCH_PLAIN, nullptr}, J, rows))) return rc;
  if ((rc = op_finish())) return rc;
  std::vector<LpRecord> rec((size_t)rows);
  D2H(rec.data(), drec, (size_t)rows * sizeof(LpRecord));
  memset(out, 0, (size_t)rows * sizeof(lnb_logprob));
  for (int i = 0; i < rows; i++) lp_finish(rec[i], out + i);
  return 0;
}

// the penalty kernels alone on host rows: logits[rows, vocab], p[rows], histories hist[rows][hist_len], pos_next[rows] -> out
extern "C" int lnb_op_penalize_f32(const float* logits, int rows, int vocab, const lnb_penalties* p, const int32_t* hist, int hist_len,
                                   const int32_t* pos_next, float* out) {
  OpScope scope_;
  if (!logits || !p || !hist || !pos_next || !out) return fail(LNB_EINVAL, "NULL argument");
  if (rows < 1 || rows > PEN_MAX_ROWS || vocab < 1 || hist_len < 1)
    return fail(LNB_EINVAL, "rows %d must be in [1, %d], vocab %d and hist_len %d >= 1", rows, PEN_MAX_ROWS, vocab, hist_len);
  int rc;
  for (int r = 0; r < rows; r++) {
    if ((rc = penalties_check(p + r, vocab))) return rc;
    if (pos_next[r] < 0 || pos_next[r] > hist_len) return fail(LNB_EINVAL, "pos_next[%d] = %d outside [0, %d]", r, pos_next[r], hist_len);
  }
  const size_t b = (size_t)rows * vocab * 4, bh = (size_t)rows * hist_len * 4;
  OPBUF(dx, b); OPBUF(dp, (size_t)rows * sizeof(lnb_penalties)); OPBUF(dh, bh); OPBUF(dc, b); OPBUF(dout, b);
  H2D(dx, logits, b);
  H2D(dp, p, (size_t)rows * sizeof(lnb_penalties));
  H2D(dh, hist, bh);
  CU(cudaMemset(dc.p, 0, b));
  PenaltyJob J{};
  J.logits = dx.as<float>(); J.ld = vocab; J.V = vocab; J.n = rows;
  J.params = dp.as<lnb_penalties>(); J.hist = dh.as<int32_t>(); J.hist_len = hist_len;
  J.cnt = dc.as<unsigned int>(); J.out = dout.as<float>(); J.pos_ptr = nullptr;
  for (int r = 0; r < rows; r++) { J.row[r] = r; J.slot[r] = r; J.seq[r] = r; J.p_next[r] = pos_next[r]; J.on[r] = lnb_pen_neutral(p + r) ? 0 : 1; }
  if ((rc = launch_penalty_job(Launcher{nullptr, LAUNCH_PLAIN, nullptr}, J))) return rc;
  if ((rc = op_finish())) return rc;
  D2H(out, dout, b);
  return 0;
}

extern "C" int lnb_op_get_rows_bf16(const uint16_t* emb, const int32_t* tokens, uint16_t* out, int S, int vocab, int dim) {
  OpScope scope_;
  if (!emb || !tokens || !out || S <= 0 || vocab <= 0 || dim <= 0 || dim % 8) return fail(LNB_EINVAL, "bad argument");
  for (int i = 0; i < S; i++)
    if (tokens[i] < 0 || tokens[i] >= vocab) return fail(LNB_EINVAL, "token id %d out of range", tokens[i]);
  OPBUF(de, (size_t)vocab * dim * 2); OPBUF(dt, (size_t)S * 4); OPBUF(dout, (size_t)S * dim * 2);
  H2D(de, emb, (size_t)vocab * dim * 2); H2D(dt, tokens, (size_t)S * 4);
  gather_rows_kernel<<<S, 256>>>(de.as<uint16_t>(), dt.as<int32_t>(), nullptr, dout.as<uint16_t>(), dim);
  int rc = op_finish();
  if (rc) return rc;
  D2H(out, dout, (size_t)S * dim * 2);
  return 0;
}
