// lnb_host.hpp -- C++ host mirror of the reference's Go packages above the C-ABI (include/lnb.h).
//
// The reference is compiled Go; the build image has no Go toolchain, so this header restates, in C++17,
// the host-side types and call sequence a Go build would keep: ml::Tensor + the ml ops on the forward
// path, model::ModelArgs / LlamaTransformer / InferenceContext, and inference::InferenceEngine with the
// generate loop of src/inference/inference.go:173-254.  Same names, argument meaning and error texts as
// the Go code (errors are exceptions instead of `(nil, error)`).  Header-only; links against liblnb.so.
#pragma once
#include <cstdint>
#include <cstring>
#include <functional>
#include <stdexcept>
#include <algorithm>
#include <cmath>
#include <memory>
#include <string>
#include <vector>

#include "../include/lnb.h"

namespace lnb_host {

struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};
inline void check(int rc) {
  if (rc < 0) throw Error(std::string("lnb: ") + lnb_last_error());
}

namespace ml {  // ---- src/ml ---------------------------------------------------------------------------
enum class DataType { BF16, F32, INT32 };  // datatype.go:11-34
inline size_t item_size(DataType t) { return t == DataType::BF16 ? 2 : 4; }

struct Tensor {  // tensor.go:11-19 (contiguous row-major, Size + RawData)
  std::vector<int> Size;
  DataType DT = DataType::BF16;
  std::vector<uint8_t> RawData;
  std::string Name;
  Tensor() = default;
  Tensor(std::vector<int> size, DataType dt) : Size(std::move(size)), DT(dt) { RawData.assign(GetElementCount() * item_size(dt), 0); }
  size_t GetElementCount() const {
    size_t n = 1;
    for (int d : Size) n *= (size_t)d;
    return n;
  }
  template <class T> T* data() { return reinterpret_cast<T*>(RawData.data()); }
  template <class T> const T* data() const { return reinterpret_cast<const T*>(RawData.data()); }
};

inline uint16_t Float32ToBFloat16bits(float f) {  // src/dtype/bfloat16.go:59-61 (truncation)
  uint32_t u;
  std::memcpy(&u, &f, 4);
  return (uint16_t)(u >> 16);
}
inline float BFloat16bitsToFloat32(uint16_t b) {  // :55-57
  uint32_t u = (uint32_t)b << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

inline int AccMode = LNB_ACC_STRICT;

inline Tensor LinearTransformation(const Tensor& input, const Tensor& weights) {  // operations_impl.go:427-447
  if (input.DT != weights.DT) throw Error("tensors are not in same data type");
  if (input.Size.size() != 2 || weights.Size.size() != 2) throw Error("LinearTransformation needs two matrices");
  if (input.Size[1] != weights.Size[1])
    throw Error("columns size " + std::to_string(input.Size[1]) + " of input tensor should be equal with " +
                std::to_string(weights.Size[1]) + " input features count of weights tensor");
  if (input.DT != DataType::BF16) throw Error("unsupported tensor datatype");
  Tensor dst({input.Size[0], weights.Size[0]}, DataType::BF16);
  check(lnb_op_linear_bf16(input.data<uint16_t>(), weights.data<uint16_t>(), dst.data<uint16_t>(), input.Size[0], input.Size[1],
                           weights.Size[0], AccMode));
  return dst;
}

inline Tensor Argmax(const Tensor& input) {  // operations_impl.go:513-548 (last dimension)
  if (input.DT != DataType::F32) throw Error("unsupported tensor datatype");
  const int cols = input.Size.back();
  const int rows = (int)(input.GetElementCount() / cols);
  Tensor dst(std::vector<int>(input.Size.begin(), input.Size.end() - 1), DataType::INT32);
  if (dst.Size.empty()) dst = Tensor({1}, DataType::INT32);
  check(lnb_op_argmax_f32(input.data<float>(), rows, cols, dst.data<int32_t>()));
  return dst;
}
}  // namespace ml

namespace model {  // ---- src/model ------------------------------------------------------------------------
struct ModelArgs : lnb_model_args {  // modelargs.go:10-44 (+ derived HeadDim / FFN width, llamatransformer.go:569-577)
  static ModelArgs Llama31_8B() {
    ModelArgs a{};
    a.dim = 4096; a.n_layers = 32; a.n_heads = 32; a.n_kv_heads = 8; a.head_dim = 128; a.ffn_dim = 14336;
    a.vocab_size = 128256; a.max_seq_len = 2048; a.norm_eps = 1e-5f; a.rope_theta = 500000.0; a.use_scaled_rope = 1;
    return a;
  }
};
struct Vocabulary {  // vocabulary.go (ids only)
  int32_t PadId = -1;
  std::vector<int32_t> StopTokenIds{128008, 128009};  // src/tiktoken/tiktokenreader.go:81
};

// src/tiktoken + model.Vocabulary's tables + the tokenizer half of src/inference/tokenize.go over lnb_vocab
struct PromptPart {  // inference.PromptPart (tokenize.go:21-25)
  std::string Header, Content;
};
class Tokenizer {
 public:
  explicit Tokenizer(const std::string& vocabFilePath) { check(lnb_vocab_load(vocabFilePath.c_str(), &h_)); }   // tiktoken.Load
  ~Tokenizer() { lnb_vocab_destroy(h_); }
  Tokenizer(const Tokenizer&) = delete;
  int Size() const { return lnb_vocab_size(h_); }
  Vocabulary GetVocabulary() const {   // PadId / StopTokenIds of NewVocabulary (vocabulary.go:23-50)
    Vocabulary v;
    int32_t stop[2];
    check(lnb_vocab_special_ids(h_, nullptr, nullptr, &v.PadId, stop));
    v.StopTokenIds = {stop[0], stop[1]};
    return v;
  }
  std::vector<int32_t> TokenizeString(const std::string& text) const {   // tokenize.go:175-193
    std::vector<int32_t> out(text.size() + 8);
    int n = 0;
    check(lnb_tokenize_string(h_, text.data(), (int64_t)text.size(), out.data(), (int)out.size(), &n));
    out.resize((size_t)n);
    return out;
  }
  std::vector<int32_t> Tokenize(const std::vector<PromptPart>& parts) const {   // tokenize.go:27-95
    std::vector<const char*> hs, cs;
    size_t cap = 32;
    for (const auto& p : parts) {
      hs.push_back(p.Header.c_str());
      cs.push_back(p.Content.c_str());
      cap += p.Header.size() + p.Content.size() + 16;
    }
    std::vector<int32_t> out(cap);
    int n = 0;
    check(lnb_tokenize_prompt(h_, hs.data(), cs.data(), (int)parts.size(), out.data(), (int)out.size(), &n));
    out.resize((size_t)n);
    return out;
  }
  // Vocabulary.IdToToken[id] (raw bytes; a piece need not be valid UTF-8)
  std::string IdToToken(int32_t id) const {
    const void* p = nullptr;
    int n = 0;
    check(lnb_vocab_token_bytes(h_, id, &p, &n));
    return std::string((const char*)p, (size_t)n);
  }
  // TokenToString (tokenize.go:195-237) without the emoji annotation: a piece that is not valid UTF-8 on its own is
  // collected in waitingBytes and released one rune per call once the bytes decode; returns addedToWaiting
  bool TokenToString(int32_t id, std::string& waitingBytes, std::string& text) const {
    const std::string piece = IdToToken(id);
    text.clear();
    if (Utf8Valid(piece)) { text = piece; return false; }
    waitingBytes += piece;
    if (!Utf8Valid(waitingBytes)) return true;
    const size_t n = Utf8RuneLen((unsigned char)waitingBytes[0]);
    text = waitingBytes.substr(0, n);
    waitingBytes.erase(0, n);
    return false;
  }
  static size_t Utf8RuneLen(unsigned char c) { return c < 0x80 ? 1 : (c >> 5) == 6 ? 2 : (c >> 4) == 14 ? 3 : 4; }
  static bool Utf8Valid(const std::string& s) {   // utf8.Valid
    for (size_t i = 0; i < s.size();) {
      const unsigned char c = (unsigned char)s[i];
      size_t n;
      uint32_t cp, min;
      if (c < 0x80) { i++; continue; }
      if ((c & 0xe0) == 0xc0) { n = 2; cp = c & 0x1f; min = 0x80; }
      else if ((c & 0xf0) == 0xe0) { n = 3; cp = c & 0x0f; min = 0x800; }
      else if ((c & 0xf8) == 0xf0) { n = 4; cp = c & 0x07; min = 0x10000; }
      else return false;
      if (i + n > s.size()) return false;
      for (size_t k = 1; k < n; k++) {
        if (((unsigned char)s[i + k] & 0xc0) != 0x80) return false;
        cp = (cp << 6) | ((unsigned char)s[i + k] & 0x3f);
      }
      if (cp < min || cp > 0x10ffff || (cp >= 0xd800 && cp <= 0xdfff)) return false;
      i += n;
    }
    return true;
  }
  std::string TokenBatchToString(const std::vector<int32_t>& ids) const {   // tokenize.go:239-258 (bytes; no emoji annotation)
    std::string out(64 + 128 * ids.size(), '\0');
    int64_t n = 0;
    int rc = lnb_detokenize(h_, ids.data(), (int)ids.size(), &out[0], (int64_t)out.size(), &n);
    if (rc != 0 && n > (int64_t)out.size()) {
      out.assign((size_t)n, '\0');
      rc = lnb_detokenize(h_, ids.data(), (int)ids.size(), &out[0], (int64_t)out.size(), &n);
    }
    check(rc);
    out.resize((size_t)n);
    return out;
  }

 private:
  lnb_vocab* h_ = nullptr;
};

class LlamaTransformer {  // llamatransformer.go:16-113
 public:
  ModelArgs args;
  LlamaTransformer(const ModelArgs& a, int device = 0) : args(a) { check(lnb_model_create(&args, device, 0, 1, nullptr, &h_)); }
  ~LlamaTransformer() { lnb_model_destroy(h_); }
  LlamaTransformer(const LlamaTransformer&) = delete;
  // getTensor + upload (loader.go:183-197)
  void UploadTensor(const std::string& name, const uint16_t* data, const std::vector<int64_t>& shape) {
    check(lnb_model_upload_tensor(h_, name.c_str(), data, shape.data(), (int)shape.size()));
  }
  void InitSynthetic(uint64_t seed) { check(lnb_model_init_synthetic(h_, seed)); }
  // torch.TorchModelReader.Load + the by-name binding of NewLlamaTransformer: checkpoint mapping -> HBM
  int LoadPth(const std::string& path) {
    int n = 0;
    check(lnb_model_load_pth(h_, path.c_str(), &n));
    return n;
  }
  // LNB_WEIGHTS_BF16, LNB_WEIGHTS_MXFP8 or LNB_WEIGHTS_MXFP4 (DESIGN §9h, §9i: Finalize quantizes the linear weights);
  // before Finalize
  void SetWeightFormat(int fmt) { check(lnb_model_set_weight_format(h_, fmt)); }
  void Finalize() { check(lnb_model_finalize(h_)); }
  // MXFP8 model: the codes [rows][cols] and scales [rows][ceil(cols / 32)] of a linear checkpoint tensor
  void MxFp8Read(const std::string& name, std::vector<uint8_t>& codes, std::vector<uint8_t>& scales, int64_t rows, int64_t cols) {
    codes.resize((size_t)(rows * cols));
    scales.resize((size_t)(rows * ((cols + 31) / 32)));
    check(lnb_model_mxfp8_read(h_, name.c_str(), codes.data(), scales.data()));
  }
  // MXFP4 model: the codes [rows][cols / 2] (the even column in a byte's low nibble) and scales [rows][ceil(cols / 32)]
  void MxFp4Read(const std::string& name, std::vector<uint8_t>& codes, std::vector<uint8_t>& scales, int64_t rows, int64_t cols) {
    codes.resize((size_t)(rows * (cols / 2)));
    scales.resize((size_t)(rows * ((cols + 31) / 32)));
    check(lnb_model_mxfp4_read(h_, name.c_str(), codes.data(), scales.data()));
  }
  struct WeightInfo {
    int Format = LNB_WEIGHTS_BF16;
    int64_t DeviceBytes = 0, StepBytes = 0;   // weight bytes in HBM; weight bytes one S = 1 step reads
  };
  WeightInfo GetWeightInfo() {
    WeightInfo w;
    check(lnb_model_weight_info(h_, &w.Format, &w.DeviceBytes, &w.StepBytes));
    return w;
  }
  lnb_model* handle() { return h_; }

 private:
  lnb_model* h_ = nullptr;
};

// src/torch: TorchModelReader over the native reader of liblnb.so (RawData aliases the read-only file mapping)
class TorchModelReader {  // torchmodelreader.go:13-66
 public:
  struct Entry {
    std::string Name;
    int DType = 0;                 // LNB_PTH_*
    std::vector<int64_t> Size;
    const void* RawData = nullptr;
    int64_t ByteCount = 0;
    bool Contiguous = true;
  };
  explicit TorchModelReader(const std::string& modelFilePath) { check(lnb_pth_open(modelFilePath.c_str(), &h_)); }
  ~TorchModelReader() { lnb_pth_close(h_); }
  TorchModelReader(const TorchModelReader&) = delete;
  std::vector<Entry> Load() const {
    std::vector<Entry> out;
    const int n = lnb_pth_tensor_count(h_);
    for (int i = 0; i < n; i++) {
      Entry e;
      const char* name = nullptr;
      int nd = 0;
      int64_t shape[8], off = 0;
      const int rc = lnb_pth_tensor_info(h_, i, &name, &e.DType, &nd, shape, &off, &e.ByteCount);
      check(rc < 0 ? rc : 0);
      e.Contiguous = (rc == 0);
      e.Name = name;
      e.Size.assign(shape, shape + nd);
      e.RawData = lnb_pth_tensor_data(h_, i);
      out.push_back(std::move(e));
    }
    return out;
  }

 private:
  lnb_pth* h_ = nullptr;
};

// loadModelArgsFromFile (modelargs.go:52-64) + derived widths; vocab_size < 1 -> rows of tok_embeddings.weight
// (the reference takes it from tokenizer.model, loader.go:103-111; the tokenizer is out of scope here)
inline ModelArgs LoadModelArgs(const std::string& modelDir, int maxSeqLen = 2048) {
  ModelArgs a{};
  check(lnb_model_args_from_params_json((modelDir + "/params.json").c_str(), maxSeqLen, &a));
  if (a.vocab_size < 1) {
    TorchModelReader r(modelDir + "/consolidated.00.pth");
    for (const auto& e : r.Load())
      if (e.Name == "tok_embeddings.weight" && !e.Size.empty()) a.vocab_size = (int32_t)e.Size[0];
    if (a.vocab_size < 1) throw Error("tensor \"tok_embeddings.weight\" not found");
  }
  return a;
}

// model.LoadModel (loader.go:18-70): <modelDir>/params.json + consolidated.00.pth -> a finalized transformer
inline std::unique_ptr<LlamaTransformer> LoadModel(const std::string& modelDir, int device = 0, int maxSeqLen = 2048,
                                                   int weightFormat = LNB_WEIGHTS_BF16) {
  auto t = std::make_unique<LlamaTransformer>(LoadModelArgs(modelDir, maxSeqLen), device);
  t->SetWeightFormat(weightFormat);
  t->LoadPth(modelDir + "/consolidated.00.pth");
  t->Finalize();
  return t;
}

// EXTENSION (the reference only has the greedy ml.Argmax): seeded sampling of the next token (lnb_session_set_sampling).
// Temperature 0 is greedy; TopK 0 is the whole vocabulary; TopP in (0, 1].
struct SamplingArgs {
  float Temperature = 0.0f;
  int32_t TopK = 0;
  float TopP = 1.0f;
  uint64_t Seed = 0;
  bool Samples() const { return Temperature != 0.0f; }
  // prompt i of a batch or continuous run samples with Seed + i (its stream is GenerateTokens' with that seed)
  SamplingArgs ForPrompt(int i) const { SamplingArgs a = *this; a.Seed += (uint64_t)i; return a; }
};

// EXTENSION: repetition, frequency and presence penalties and a logit bias over the sequence's token history
// (lnb_session_set_penalties, DESIGN.md §9e).  The defaults are neutral (off).  CountPrompt false counts generated tokens only:
// first_pos is the prompt's length.  A -inf bias bans its token.
struct PenaltyArgs {
  float RepetitionPenalty = 1.0f;
  float FrequencyPenalty = 0.0f;
  float PresencePenalty = 0.0f;
  int32_t Window = 0;          // the last Window positions; 0: all
  bool CountPrompt = false;
  std::vector<std::pair<int32_t, float>> LogitBias;
  bool Neutral() const { return RepetitionPenalty == 1.0f && FrequencyPenalty == 0.0f && PresencePenalty == 0.0f && LogitBias.empty(); }
  lnb_penalties C(int promptLength) const {
    if (LogitBias.size() > LNB_LOGIT_BIAS_MAX) throw Error("LogitBias has more than " + std::to_string(LNB_LOGIT_BIAS_MAX) + " entries");
    lnb_penalties p{};
    p.repetition_penalty = RepetitionPenalty;
    p.frequency_penalty = FrequencyPenalty;
    p.presence_penalty = PresencePenalty;
    p.window = Window;
    p.first_pos = CountPrompt ? 0 : promptLength;
    p.n_bias = (int32_t)LogitBias.size();
    for (size_t j = 0; j < LogitBias.size(); j++) { p.bias_token[j] = LogitBias[j].first; p.bias[j] = LogitBias[j].second; }
    return p;
  }
};

// EXTENSION: speculative decoding (lnb_forward_speculative) with prompt-lookup drafts of up to MaxDraft tokens.  Branches > 1:
// trees of up to MaxDraft nodes holding the top Branches continuations (PromptLookupTree, lnb_forward_speculative_tree); not
// with penalties, a grammar or logprobs
struct SpeculativeArgs {
  int MaxDraft = 0;
  int NgramMax = 3;
  int NgramMin = 1;
  int Branches = 1;
};

// Prompt-lookup drafter (the Python mirror's prompt_lookup_drafts), a pure function of the history h[0..L) whose last token
// is about to be fed: for n = ngramMax down to ngramMin, the largest j with j + n < L and h[j..j+n) == h[L-n..L); the first n
// that matches gives the drafts h[j+n .. min(j+n+maxDraft, L)).  No match gives no drafts.
inline std::vector<int32_t> PromptLookupDrafts(const std::vector<int32_t>& h, int maxDraft, int ngramMax = 3, int ngramMin = 1) {
  const int L = (int)h.size();
  if (maxDraft <= 0) return {};
  for (int n = ngramMax; n >= std::max(ngramMin, 1); n--) {
    if (L < n + 1) continue;
    for (int j = L - n - 1; j >= 0; j--) {
      if (!std::equal(h.begin() + j, h.begin() + j + n, h.begin() + (L - n))) continue;
      return std::vector<int32_t>(h.begin() + j + n, h.begin() + std::min(j + n + maxDraft, L));
    }
  }
  return {};
}

// Tree drafter (the Python mirror's prompt_lookup_tree), a pure function of the history: up to `branches` distinct
// continuations h[j+n .. min(j+n+maxNodes, L)), for n = ngramMax down to ngramMin and within one n the matches from the most
// recent; merged into a trie under the root (row 0), numbered breadth first (a depth's nodes in the order of the first
// continuation that reaches them) and cut to maxNodes.  tokens[i] / parents[i]: node i is row i + 1 under row parents[i].
// branches = 1 gives PromptLookupDrafts as a chain.
inline void PromptLookupTree(const std::vector<int32_t>& h, int maxNodes, int branches, int ngramMax, int ngramMin,
                             std::vector<int32_t>& tokens, std::vector<int32_t>& parents) {
  tokens.clear();
  parents.clear();
  const int L = (int)h.size();
  if (maxNodes <= 0 || branches <= 0) return;
  std::vector<std::vector<int32_t>> conts;
  for (int n = ngramMax; n >= std::max(ngramMin, 1) && (int)conts.size() < branches; n--) {
    if (L < n + 1) continue;
    for (int j = L - n - 1; j >= 0 && (int)conts.size() < branches; j--) {
      if (!std::equal(h.begin() + j, h.begin() + j + n, h.begin() + (L - n))) continue;
      std::vector<int32_t> c(h.begin() + j + n, h.begin() + std::min(j + n + maxNodes, L));
      if (std::find(conts.begin(), conts.end(), c) == conts.end()) conts.push_back(c);
    }
  }
  // trie nodes as (depth, rank of the first continuation reaching it, that continuation): breadth first, then rank
  std::vector<std::pair<std::pair<int, int>, std::vector<int32_t>>> nodes;
  for (int r = 0; r < (int)conts.size(); r++)
    for (int d = 1; d <= (int)conts[r].size(); d++) {
      std::vector<int32_t> key(conts[r].begin(), conts[r].begin() + d);
      bool seen = false;
      for (const auto& nd : nodes) seen |= nd.second == key;
      if (!seen) nodes.push_back({{d, r}, key});
    }
  std::stable_sort(nodes.begin(), nodes.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  if ((int)nodes.size() > maxNodes) nodes.resize((size_t)maxNodes);
  for (size_t i = 0; i < nodes.size(); i++) {
    const std::vector<int32_t>& key = nodes[i].second;
    int par = 0;
    for (size_t k = 0; k < i; k++)
      if (nodes[k].second.size() + 1 == key.size() && std::equal(key.begin(), key.end() - 1, nodes[k].second.begin())) par = (int)k + 1;
    tokens.push_back(key.back());
    parents.push_back(par);
  }
}

// EXTENSION: regex-constrained generation (lnb_grammar_create, DESIGN.md §9g).  The tokens a sequence emits after the
// grammar's first position spell a prefix of a string of re.fullmatch(regex, s, re.ASCII); a stop token (Z: the
// tokenizer's stop ids) only follows a complete match.  Token bytes come from the tokenizer, special tokens are empty.  The
// masks of every state are built on the model's device, once.
class Grammar {
 public:
  Grammar(LlamaTransformer& t, const std::string& regex, const Tokenizer& tok) {
    const int V = t.args.vocab_size, nMerge = tok.Size() - 256;
    std::vector<uint8_t> bytes;
    std::vector<int64_t> off(1, 0);
    for (int i = 0; i < V; i++) {
      if (i < nMerge) {
        const std::string b = tok.IdToToken(i);
        bytes.insert(bytes.end(), b.begin(), b.end());
      }
      off.push_back((int64_t)bytes.size());
    }
    const std::vector<int32_t> stop = tok.GetVocabulary().StopTokenIds;
    check(lnb_grammar_create(t.handle(), regex.data(), (int64_t)regex.size(), bytes.data(), off.data(), stop.data(), (int)stop.size(), &h_));
  }
  ~Grammar() { lnb_grammar_destroy(h_); }
  Grammar(const Grammar&) = delete;
  const lnb_grammar* handle() const { return h_; }

 private:
  lnb_grammar* h_ = nullptr;
};

class InferenceContext {  // inferencecontext.go:8-46 (KV cache in HBM)
 public:
  int SequenceLength;
  InferenceContext(LlamaTransformer& t, int sequenceLength, int accMode = LNB_ACC_STRICT, int maxRows = 8)
      : SequenceLength(sequenceLength > 0 ? sequenceLength : t.args.max_seq_len), vocab_(t.args.vocab_size), maxRows_(maxRows) {
    check(lnb_session_create(t.handle(), SequenceLength, maxRows, accMode, &h_));
  }
  // n reference InferenceContexts that share the weights (batched decode): own KV cache and position each
  InferenceContext(LlamaTransformer& t, int sequenceLength, int accMode, int maxRows, int nSeq)
      : SequenceLength(sequenceLength > 0 ? sequenceLength : t.args.max_seq_len), vocab_(t.args.vocab_size),
        maxRows_(std::max(maxRows, nSeq)) {
    check(lnb_session_create_batch(t.handle(), SequenceLength, nSeq, maxRows, accMode, &h_));
  }
  // the same with the KV cache in format kvFormat (LNB_KV_BF16 or LNB_KV_MXFP8, lnb_session_create_kv; nSeq 1..8)
  InferenceContext(LlamaTransformer& t, int sequenceLength, int accMode, int maxRows, int nSeq, int kvFormat)
      : SequenceLength(sequenceLength > 0 ? sequenceLength : t.args.max_seq_len), vocab_(t.args.vocab_size),
        maxRows_(nSeq > 1 ? std::max(maxRows, nSeq) : maxRows) {
    check(lnb_session_create_kv(t.handle(), SequenceLength, nSeq, maxRows, accMode, kvFormat, &h_));
  }
  ~InferenceContext() { lnb_session_destroy(h_); }
  void SetActiveSequence(int seq) { check(lnb_session_set_active_sequence(h_, seq)); }
  // sequence seq samples its next tokens with *a (nullptr or Temperature 0: greedy); the token outputs below then carry them
  void SetSampling(int seq, const SamplingArgs* a) {
    if (!a || !a->Samples()) { check(lnb_session_set_sampling(h_, seq, nullptr)); return; }
    const lnb_sampling p{a->Temperature, a->TopK, a->TopP, a->Seed};
    check(lnb_session_set_sampling(h_, seq, &p));
  }
  // EXTENSION: sequence seq is penalized with *a (nullptr or neutral: off) for a prompt of promptLength tokens; turning
  // penalties on clears its token history
  void SetPenalties(int seq, const PenaltyArgs* a, int promptLength) {
    if (!a) { check(lnb_session_set_penalties(h_, seq, nullptr)); return; }
    const lnb_penalties p = a->C(promptLength);
    check(lnb_session_set_penalties(h_, seq, &p));
  }
  // EXTENSION: sequence seq is constrained by *g (nullptr: off) from its next forward on, its grammar starting at position
  // firstPos (typically the prompt's length)
  void SetGrammar(int seq, const Grammar* g, int firstPos) { check(lnb_session_set_grammar(h_, seq, g ? g->handle() : nullptr, firstPos)); }
  // EXTENSION: token log-probabilities (lnb_session_set_logprobs).  topN 0..20 turns them on for sequence seq, -1 off; every
  // token the context then emits for seq writes the record of the position it occupies (the raw model distribution).
  void SetLogprobs(int seq, int topN) { check(lnb_session_set_logprobs(h_, seq, topN)); }
  // records [pos0, pos0 + n) of sequence seq (token -1: never written)
  std::vector<lnb_logprob> ReadLogprobs(int seq, int pos0, int n) {
    std::vector<lnb_logprob> out((size_t)n);
    check(lnb_session_logprobs_read(h_, seq, pos0, n, out.data()));
    return out;
  }
  // lnb_score: the log-probability of tokens[1..] given what precedes them, one forward of the active sequence over
  // tokens[0 .. n-1) at startPos -> the records of positions startPos + 1 .. startPos + n - 1
  std::vector<lnb_logprob> Score(const std::vector<int32_t>& tokens, int startPos, int seq = 0) {
    check(lnb_score(h_, tokens.data(), (int)tokens.size(), startPos));
    return ReadLogprobs(seq, startPos + 1, (int)tokens.size() - 1);
  }
  // Forward + last-row ml.Argmax in one call (inference.go:202-216), 4-byte read-back
  int32_t ForwardArgmax(const std::vector<int32_t>& tokens, int startPos) {
    int32_t next = -1;
    check(lnb_forward(h_, tokens.data(), (int)tokens.size(), startPos, nullptr, 0, &next));
    return next;
  }
  // one decode step of every sequence: tokens[i] at positions[i] -> greedy next token of sequence i
  std::vector<int32_t> ForwardBatch(const std::vector<int32_t>& tokens, const std::vector<int32_t>& positions) {
    std::vector<int32_t> next(tokens.size(), -1);
    check(lnb_forward_batch(h_, tokens.data(), positions.data(), (int)tokens.size(), nullptr, next.data()));
    return next;
  }
  // EXTENSION (continuous batching, lnb_forward_ragged): ONE forward over segments of different sequences, each with the
  // arithmetic of its own Forward -> greedy token of each segment's last row
  struct Segment { int seq, startPos; std::vector<int32_t> tokens; };
  std::vector<int32_t> ForwardRagged(const std::vector<Segment>& segs) {
    std::vector<int32_t> seq, start, len, flat, next(segs.size(), -1);
    for (const Segment& s : segs) {
      seq.push_back(s.seq);
      start.push_back(s.startPos);
      len.push_back((int32_t)s.tokens.size());
      flat.insert(flat.end(), s.tokens.begin(), s.tokens.end());
    }
    check(lnb_forward_ragged(h_, (int)segs.size(), seq.data(), start.data(), len.data(), flat.data(), nullptr, next.data()));
    return next;
  }
  // EXTENSION (speculative verification, lnb_forward_speculative): segment tokens = the sequence's last emitted token + drafts,
  // row j at startPos + j.  -> next token of every row; accepted[i] = drafts of segment i the model agrees with (segment i
  // emits the next tokens of its rows 0 .. accepted[i])
  std::vector<int32_t> ForwardSpeculative(const std::vector<Segment>& segs, std::vector<int32_t>& accepted) {
    std::vector<int32_t> seq, start, n_draft, flat;
    for (const Segment& s : segs) {
      seq.push_back(s.seq);
      start.push_back(s.startPos);
      n_draft.push_back((int32_t)s.tokens.size() - 1);
      flat.insert(flat.end(), s.tokens.begin(), s.tokens.end());
    }
    std::vector<int32_t> next(flat.size(), -1);
    accepted.assign(segs.size(), 0);
    check(lnb_forward_speculative(h_, (int)segs.size(), seq.data(), start.data(), n_draft.data(), flat.data(), nullptr, next.data(),
                                  accepted.data()));
    return next;
  }
  // EXTENSION (tree verification, lnb_forward_speculative_tree): segment tokens = the sequence's last emitted token + the
  // nodes, parents[s][j] the parent row of row j (parents[s][0] is not read).  -> next token of every row; accepted[i] = the
  // depth segment i reaches, paths[i] = its accepted rows, segment-local, root first (segment i emits their next tokens)
  std::vector<int32_t> ForwardSpeculativeTree(const std::vector<Segment>& segs, const std::vector<std::vector<int32_t>>& parents,
                                              std::vector<int32_t>& accepted, std::vector<std::vector<int32_t>>& paths) {
    std::vector<int32_t> seq, start, n_nodes, flat, par;
    for (size_t k = 0; k < segs.size(); k++) {
      const Segment& s = segs[k];
      if (parents[k].size() != s.tokens.size()) throw Error("a tree segment needs one parent entry per row");
      seq.push_back(s.seq);
      start.push_back(s.startPos);
      n_nodes.push_back((int32_t)s.tokens.size() - 1);
      flat.insert(flat.end(), s.tokens.begin(), s.tokens.end());
      par.insert(par.end(), parents[k].begin(), parents[k].end());
    }
    std::vector<int32_t> next(flat.size(), -1), path(flat.size(), -1);
    accepted.assign(segs.size(), 0);
    check(lnb_forward_speculative_tree(h_, (int)segs.size(), seq.data(), start.data(), n_nodes.data(), par.data(), flat.data(), nullptr,
                                       next.data(), accepted.data(), path.data()));
    paths.assign(segs.size(), {});
    for (size_t k = 0, w = 0, r0 = 0; k < segs.size(); r0 += segs[k].tokens.size(), k++)
      for (int d = 0; d <= accepted[k]; d++) paths[k].push_back(path[w++] - (int32_t)r0);
    return next;
  }
  // EXTENSION (lnb_session_copy_sequences): positions [pos0, pos1) of sequence dst[i] get what sequence src[i] held there
  // before the call (K and V of every layer, the penalty history, the logprob records); the sources are read as a snapshot
  void CopySequences(const std::vector<int32_t>& src, const std::vector<int32_t>& dst, int pos0, int pos1) {
    if (src.size() != dst.size()) throw Error(std::to_string(src.size()) + " sources for " + std::to_string(dst.size()) + " destinations");
    check(lnb_session_copy_sequences(h_, (int)src.size(), src.data(), dst.data(), pos0, pos1));
  }
  int MaxRows() const { return maxRows_; }
  InferenceContext(const InferenceContext&) = delete;
  // LlamaTransformer.Forward (llamatransformer.go:145-180): tokens [S] -> f32 logits [S, vocab]
  ml::Tensor Forward(const ml::Tensor& inputTokens, int startPos) {
    if (inputTokens.DT != ml::DataType::INT32 || inputTokens.Size.size() != 1) throw Error("inputTokens must be a 1-D Int32 tensor");
    const int S = inputTokens.Size[0];
    if (S == 0) throw Error("empty token array");
    ml::Tensor logits({S, vocab_}, ml::DataType::F32);
    check(lnb_forward(h_, inputTokens.data<int32_t>(), S, startPos, logits.data<float>(), 1, nullptr));
    return logits;
  }
  // The same Forward with the logits left in HBM (lnb_forward_device): the returned handle stands for the [rowsKept, vocab]
  // tensor; ArgmaxRows = Slice + ml.Argmax on the device (4 bytes per row back), ReadLogits = touching the tensor's data.
  // A handle is valid until the context's next forward.
  struct DeviceLogits { int64_t generation = 0; int rows = 0; };
  DeviceLogits ForwardDevice(const std::vector<int32_t>& tokens, int startPos, bool allRows = false, int32_t* argmaxLast = nullptr) {
    DeviceLogits d;
    d.rows = allRows ? (int)tokens.size() : 1;
    check(lnb_forward_device(h_, tokens.data(), (int)tokens.size(), startPos, d.rows, argmaxLast, &d.generation));
    return d;
  }
  std::vector<int32_t> ArgmaxRows(const DeviceLogits& d, int row0, int rows) {
    std::vector<int32_t> out((size_t)rows, -1);
    check(lnb_session_logits_argmax(h_, d.generation, row0, rows, out.data()));
    return out;
  }
  ml::Tensor ReadLogits(const DeviceLogits& d, int row0, int rows) {
    ml::Tensor t({rows, vocab_}, ml::DataType::F32);
    check(lnb_session_logits_read(h_, d.generation, row0, rows, t.data<float>()));
    return t;
  }
  // chunked prefill (EXTENSION, SURVEY 8f-4): allow S > 1 calls at startPos > 0 with the [S,T] causal mask
  void AllowChunkedPrefill(bool on) { check(lnb_session_set_chunked_prefill(h_, on ? 1 : 0)); }
  // 1 = the persistent decode engine serves this context's S=1 calls, 0 = the kernel chain
  bool UsesDecodeEngine() { return lnb_session_decode_engine(h_) == 1; }
  // after LNB_ETIMEOUT on the peer all-reduce: back to ncclAllReduce (every rank must do the same)
  void DisablePeerAllReduce() { check(lnb_session_p2p_disable(h_)); }
  lnb_session* handle() { return h_; }

 private:
  lnb_session* h_ = nullptr;
  int vocab_;
  int maxRows_;
};
}  // namespace model

namespace inference {  // ---- src/inference ------------------------------------------------------------------
enum GenerationState { GSInProgress = 0, GSFinishedByReachingEOS = 1, GSFinishedByReachingSeqLen = 2 };

// speculative trees (Branches > 1) key nothing by position: not with penalties, a grammar or logprobs (keyed)
inline void CheckSpeculativeTree(const model::SpeculativeArgs* spec, bool keyed) {
  if (spec && spec->Branches < 1) throw Error("SpeculativeArgs.Branches must be >= 1");
  if (spec && spec->Branches > 1 && keyed)
    throw Error("speculative trees (Branches > 1) with penalties, a grammar or logprobs are not built: their records are keyed by "
                "position, which sibling drafts share");
}

// The speculative loop of the Python mirror's _generate_speculative: hists[i] = the tokens of sequence i so far, its last one
// emitted and fed next (at position size - 1); every live sequence gets a row per call, the rest of min(8, maxRows) rows go to
// prompt-lookup drafts in sequence order, no row past position SequenceLength - 2; the accepted tokens are emitted one at a
// time through the stop logic of generateTokensInternal (inference.go:218-248).  emit(sequence, state, token).
inline void GenerateSpeculative(model::InferenceContext& infContext, const model::Vocabulary& vocab,
                                std::vector<std::vector<int32_t>>& hists, std::vector<int> live, const model::SpeculativeArgs& spec,
                                const std::function<void(int, GenerationState, int32_t)>& emit,
                                std::vector<std::vector<lnb_logprob>>* logprobsOut = nullptr) {
  const int seqLen = infContext.SequenceLength;
  const int budget = std::min(8, infContext.MaxRows());
  const bool tree = spec.Branches > 1;
  if ((int)live.size() > budget) throw Error("more live sequences than rows in a speculative call");
  while (!live.empty()) {
    int left = budget - (int)live.size();
    std::vector<model::InferenceContext::Segment> segs;
    std::vector<std::vector<int32_t>> parents;
    for (int i : live) {
      const int pos = (int)hists[i].size() - 1;
      const int k = std::min({spec.MaxDraft, left, seqLen - 2 - pos});
      std::vector<int32_t> toks{hists[i].back()}, d, par{-1};
      if (tree) model::PromptLookupTree(hists[i], k, spec.Branches, spec.NgramMax, spec.NgramMin, d, par);
      else d = model::PromptLookupDrafts(hists[i], k, spec.NgramMax, spec.NgramMin);
      if (tree) par.insert(par.begin(), -1);
      left -= (int)d.size();
      toks.insert(toks.end(), d.begin(), d.end());
      segs.push_back({i, pos, toks});
      parents.push_back(par);
    }
    std::vector<int32_t> accepted;
    std::vector<std::vector<int32_t>> paths;
    const std::vector<int32_t> next =
        tree ? infContext.ForwardSpeculativeTree(segs, parents, accepted, paths) : infContext.ForwardSpeculative(segs, accepted);
    if (!tree)
      for (int32_t a : accepted) {
        paths.emplace_back();
        for (int d = 0; d <= a; d++) paths.back().push_back(d);
      }
    std::vector<int> still;
    int r0 = 0;
    for (size_t k = 0; k < segs.size(); k++) {
      const int i = segs[k].seq;
      bool finished = false;
      std::vector<lnb_logprob> recs;   // the records of the accepted positions
      if (logprobsOut) recs = infContext.ReadLogprobs(i, segs[k].startPos + 1, accepted[k] + 1);
      for (int j = 0; j <= accepted[k] && !finished; j++) {
        const int32_t tok = next[r0 + paths[k][(size_t)j]];
        const int curPos = segs[k].startPos + 1 + j;
        hists[i].push_back(tok);
        if (logprobsOut) (*logprobsOut)[(size_t)i].push_back(recs[(size_t)j]);
        bool eos = false;
        for (int32_t s : vocab.StopTokenIds) eos |= (s == tok);
        const GenerationState st = eos ? GSFinishedByReachingEOS : (curPos + 1 == seqLen ? GSFinishedByReachingSeqLen : GSInProgress);
        emit(i, st, tok);
        finished = st != GSInProgress;
      }
      r0 += (int)segs[k].tokens.size();
      if (!finished) still.push_back(i);
    }
    live = still;
  }
}

// generateTokensInternal (inference.go:173-254); `emit` plays generatedTokensCh.  EXTENSION: logprobs 0..20 turns on token
// log-probabilities; logprobsOut (or nullptr) then gets one record per emitted token, in order.  penalties (or nullptr):
// every emitted token is drawn from the penalized logits (the records stay the raw distribution's).  grammar (or nullptr):
// every emitted token is one the grammar allows after the tokens emitted before it.
inline void GenerateTokens(model::LlamaTransformer& transformer, const model::Vocabulary& vocab, int sequenceLength, int accMode,
                           const std::vector<int32_t>& promptTokens, const std::function<void(GenerationState, int32_t)>& emit,
                           const model::SamplingArgs* sampling = nullptr, const model::SpeculativeArgs* speculative = nullptr,
                           int logprobs = -1, std::vector<lnb_logprob>* logprobsOut = nullptr,
                           const model::PenaltyArgs* penalties = nullptr, const model::Grammar* grammar = nullptr) {
  // the prefill call carries the whole prompt: size the session's row buffers for it
  model::InferenceContext infContext(transformer, sequenceLength, accMode, std::max<int>(8, (int)promptTokens.size()));
  if (penalties && penalties->Neutral()) penalties = nullptr;
  CheckSpeculativeTree(speculative, penalties || grammar || logprobs >= 0);
  const bool samples = (sampling && sampling->Samples()) || penalties || grammar;
  if (sampling && sampling->Samples()) infContext.SetSampling(0, sampling);   // the sampled token instead of Slice + ml.Argmax
  if (penalties) infContext.SetPenalties(0, penalties, (int)promptTokens.size());
  if (grammar) infContext.SetGrammar(0, grammar, (int)promptTokens.size());
  if (logprobs >= 0) infContext.SetLogprobs(0, logprobs);
  if (logprobs < 0) logprobsOut = nullptr;
  const int promptLength = (int)promptTokens.size();
  if (promptLength >= infContext.SequenceLength)
    throw Error("context SequenceLength " + std::to_string(infContext.SequenceLength) + " must be higher than prompt tokens length " +
                std::to_string(promptLength));
  std::vector<int32_t> tokens(infContext.SequenceLength, vocab.PadId);  // ml.Full(..., PadId) :181
  std::copy(promptTokens.begin(), promptTokens.end(), tokens.begin());
  int prevPos = 0;
  for (int curPos = promptLength; curPos < infContext.SequenceLength; curPos++) {  // :194
    int32_t nextTokenId;
    if (samples) {
      nextTokenId = infContext.ForwardArgmax(std::vector<int32_t>(tokens.begin() + prevPos, tokens.begin() + curPos), prevPos);
    } else {
      ml::Tensor slice({curPos - prevPos}, ml::DataType::INT32);                   // tokens.Slice([prevPos],[curPos]) :195
      std::memcpy(slice.RawData.data(), tokens.data() + prevPos, (size_t)(curPos - prevPos) * 4);
      ml::Tensor logits = infContext.Forward(slice, prevPos);                      // :202
      const int rows = logits.Size[0], V = logits.Size[1];
      ml::Tensor last({1, V}, ml::DataType::F32);                                  // logits.Slice(last row) :207
      std::memcpy(last.RawData.data(), logits.data<float>() + (size_t)(rows - 1) * V, (size_t)V * 4);
      nextTokenId = ml::Argmax(last).data<int32_t>()[0];                           // :211
    }
    if (tokens[curPos] != vocab.PadId) nextTokenId = tokens[curPos];               // :218-226
    tokens[curPos] = nextTokenId;
    if (logprobsOut) logprobsOut->push_back(infContext.ReadLogprobs(0, curPos, 1)[0]);
    bool eos = false;
    for (int32_t s : vocab.StopTokenIds) eos |= (s == nextTokenId);
    prevPos = curPos;
    if (eos) { emit(GSFinishedByReachingEOS, nextTokenId); break; }                 // :233-240
    if (curPos + 1 == infContext.SequenceLength) { emit(GSFinishedByReachingSeqLen, nextTokenId); break; }
    emit(GSInProgress, nextTokenId);
    if (speculative) {   // EXTENSION: the prompt is in the cache; from here on every call verifies drafts (same stream)
      std::vector<std::vector<int32_t>> hists{std::vector<int32_t>(tokens.begin(), tokens.begin() + curPos + 1)};
      std::vector<std::vector<lnb_logprob>> lp(1);
      GenerateSpeculative(infContext, vocab, hists, {0}, *speculative, [&](int, GenerationState st, int32_t tok) { emit(st, tok); },
                          logprobsOut ? &lp : nullptr);
      if (logprobsOut) logprobsOut->insert(logprobsOut->end(), lp[0].begin(), lp[0].end());
      break;
    }
  }
}

// The consumer InferenceEngine.TokenizeBatch (src/inference/tokenize.go:97-107) never got in the reference
// (SURVEY 8f-4): every prompt runs the loop above -- own KV cache, positions and stop condition -- but all
// sequences advance together, one pass over the weights per step.  emit(sequence, state, token).  logprobs / logprobsOut as in
// GenerateTokens, one list per prompt; penalties and grammar as in GenerateTokens, for every sequence.
inline void GenerateTokensBatch(model::LlamaTransformer& transformer, const model::Vocabulary& vocab, int sequenceLength, int accMode,
                                const std::vector<std::vector<int32_t>>& prompts,
                                const std::function<void(int, GenerationState, int32_t)>& emit,
                                const model::SamplingArgs* sampling = nullptr, const model::SpeculativeArgs* speculative = nullptr,
                                int logprobs = -1, std::vector<std::vector<lnb_logprob>>* logprobsOut = nullptr,
                                const model::PenaltyArgs* penalties = nullptr, const model::Grammar* grammar = nullptr) {
  const int n = (int)prompts.size();
  if (n < 1) throw Error("empty prompt batch");
  CheckSpeculativeTree(speculative, (penalties && !penalties->Neutral()) || grammar || logprobs >= 0);
  model::InferenceContext infContext(transformer, sequenceLength, accMode, std::max(8, n), n);
  if (penalties)
    for (int i = 0; i < n; i++) infContext.SetPenalties(i, penalties, (int)prompts[i].size());
  if (grammar)
    for (int i = 0; i < n; i++) infContext.SetGrammar(i, grammar, (int)prompts[i].size());
  if (logprobs >= 0)
    for (int i = 0; i < n; i++) infContext.SetLogprobs(i, logprobs);
  if (logprobs < 0) logprobsOut = nullptr;
  if (logprobsOut) logprobsOut->assign((size_t)n, {});
  if (sampling && sampling->Samples())
    for (int i = 0; i < n; i++) {
      const model::SamplingArgs a = sampling->ForPrompt(i);
      infContext.SetSampling(i, &a);
    }
  const int seqLen = infContext.SequenceLength;
  for (const auto& p : prompts)
    if ((int)p.size() >= seqLen)
      throw Error("context SequenceLength " + std::to_string(seqLen) + " must be higher than prompt tokens length " + std::to_string(p.size()));
  std::vector<int32_t> cur(n), pos(n);
  std::vector<char> done(n, 0);
  int n_done = 0;
  auto record = [&](int i, int32_t tok, int curPos) {   // :218-248
    cur[i] = tok;
    pos[i] = curPos;
    if (logprobsOut) (*logprobsOut)[(size_t)i].push_back(infContext.ReadLogprobs(i, curPos, 1)[0]);
    bool eos = false;
    for (int32_t s : vocab.StopTokenIds) eos |= (s == tok);
    GenerationState st = eos ? GSFinishedByReachingEOS : (curPos + 1 == seqLen ? GSFinishedByReachingSeqLen : GSInProgress);
    if (st != GSInProgress) { done[i] = 1; n_done++; }
    emit(i, st, tok);
  };
  for (int i = 0; i < n; i++) {                           // prefill on sequence i's cache
    infContext.SetActiveSequence(i);
    record(i, infContext.ForwardArgmax(prompts[i], 0), (int)prompts[i].size());
  }
  if (speculative) {   // EXTENSION: one lnb_forward_speculative per call, a row per unfinished sequence, drafts in the rest
    std::vector<std::vector<int32_t>> hists(n);
    std::vector<int> live;
    for (int i = 0; i < n; i++) {
      hists[i] = prompts[i];
      hists[i].push_back(cur[i]);
      if (!done[i]) live.push_back(i);
    }
    GenerateSpeculative(infContext, vocab, hists, live, *speculative, emit, logprobsOut);
    return;
  }
  while (n_done < n) {
    // finished sequences are stepped again at their last position (a no-op for their state)
    const std::vector<int32_t> next = infContext.ForwardBatch(cur, pos);
    for (int i = 0; i < n; i++)
      if (!done[i]) record(i, next[i], pos[i] + 1);
  }
}

// Continuous batching (EXTENSION, lnb_forward_ragged): any number of prompts through at most `slots` live sequences, the
// scheduler of the Python mirror's GenerateTokensContinuous.  Every step is ONE forward: each decoding sequence gets its
// row, the rest of the stepTokens-row budget goes to prompt chunks first in first out, a prompt whose last chunk is in the
// step emits its first token, a finished slot takes the next waiting prompt at position 0; steps without prompt rows run
// lnb_forward_batch.  emit(prompt index, state, token); per prompt the stream is GenerateTokens' own.  logprobs / logprobsOut
// as in GenerateTokens, one list per prompt; penalties and grammar as in GenerateTokens, set at each admission (first_pos
// follows the prompt).
inline void GenerateTokensContinuous(model::LlamaTransformer& transformer, const model::Vocabulary& vocab, int sequenceLength,
                                     int accMode, const std::vector<std::vector<int32_t>>& prompts, int slots, int stepTokens,
                                     const std::function<void(int, GenerationState, int32_t)>& emit,
                                     const model::SamplingArgs* sampling = nullptr, int logprobs = -1,
                                     std::vector<std::vector<lnb_logprob>>* logprobsOut = nullptr,
                                     const model::PenaltyArgs* penalties = nullptr, const model::Grammar* grammar = nullptr) {
  if (slots < 1 || slots > 8) throw Error("slots must be in [1, 8]");
  if (stepTokens < slots) throw Error("stepTokens must be at least slots (every decoding sequence gets a row)");
  model::InferenceContext infContext(transformer, sequenceLength, accMode, std::max(8, stepTokens), slots);
  const int seqLen = infContext.SequenceLength, budget = std::min(stepTokens, infContext.MaxRows());
  for (const auto& p : prompts)
    if (p.empty() || (int)p.size() >= seqLen)
      throw Error("context SequenceLength " + std::to_string(seqLen) + " must be higher than prompt tokens length " + std::to_string(p.size()) +
                  " (and prompts must not be empty)");
  if (logprobs >= 0)
    for (int k = 0; k < slots; k++) infContext.SetLogprobs(k, logprobs);
  if (logprobs < 0) logprobsOut = nullptr;
  if (logprobsOut) logprobsOut->assign(prompts.size(), {});
  struct Slot { int i = -1, fed = 0, order = 0; int32_t cur = -1; int pos = 0; bool decoding = false; };
  std::vector<Slot> slot((size_t)slots);
  size_t next_prompt = 0;
  int admitted = 0, live = 0;
  while (next_prompt < prompts.size() || live > 0) {
    for (Slot& s : slot)
      if (s.i < 0 && next_prompt < prompts.size()) {
        s = Slot(); s.i = (int)next_prompt++; s.order = admitted++; live++;
        if (sampling && sampling->Samples()) {   // before the prompt's first segment
          const model::SamplingArgs a = sampling->ForPrompt(s.i);
          infContext.SetSampling((int)(&s - slot.data()), &a);
        }
        if (penalties) infContext.SetPenalties((int)(&s - slot.data()), penalties, (int)prompts[(size_t)s.i].size());
        if (grammar) infContext.SetGrammar((int)(&s - slot.data()), grammar, (int)prompts[(size_t)s.i].size());
      }
    std::vector<int> decoding, prefilling;
    for (int k = 0; k < slots; k++)
      if (slot[k].i >= 0) (slot[k].decoding ? decoding : prefilling).push_back(k);
    std::sort(prefilling.begin(), prefilling.end(), [&](int a, int b) { return slot[a].order < slot[b].order; });
    std::vector<model::InferenceContext::Segment> segs;
    std::vector<int> seg_slot;
    for (int k : decoding) { segs.push_back({k, slot[k].pos, {slot[k].cur}}); seg_slot.push_back(k); }
    int left = budget - (int)decoding.size();
    for (int k : prefilling) {
      if (left <= 0) break;
      const std::vector<int32_t>& p = prompts[(size_t)slot[k].i];
      const int n = std::min(left, (int)p.size() - slot[k].fed);
      segs.push_back({k, slot[k].fed, std::vector<int32_t>(p.begin() + slot[k].fed, p.begin() + slot[k].fed + n)});
      seg_slot.push_back(k);
      left -= n;
    }
    std::vector<int32_t> out((size_t)slots, -1);
    if (prefilling.empty()) {   // decode rows only: one batch-engine launch, row k = slot k (free slots: token 0 at 0)
      const int n = decoding.back() + 1;
      std::vector<int32_t> toks((size_t)n, 0), poss((size_t)n, 0);
      for (int k : decoding) { toks[(size_t)k] = slot[k].cur; poss[(size_t)k] = slot[k].pos; }
      const std::vector<int32_t> next = infContext.ForwardBatch(toks, poss);
      for (int k : decoding) out[(size_t)k] = next[(size_t)k];
    } else {
      const std::vector<int32_t> next = infContext.ForwardRagged(segs);
      for (size_t j = 0; j < segs.size(); j++) out[(size_t)seg_slot[j]] = next[j];
    }
    for (size_t j = 0; j < segs.size(); j++) {
      Slot& s = slot[(size_t)seg_slot[j]];
      int curPos;
      if (!s.decoding) {
        s.fed += (int)segs[j].tokens.size();
        if (s.fed < (int)prompts[(size_t)s.i].size()) continue;
        curPos = s.fed;
        s.decoding = true;
      } else {
        curPos = s.pos + 1;
      }
      const int32_t tok = out[(size_t)seg_slot[j]];
      s.cur = tok;
      s.pos = curPos;
      bool eos = false;
      for (int32_t st : vocab.StopTokenIds) eos |= (st == tok);
      const GenerationState state = eos ? GSFinishedByReachingEOS : (curPos + 1 == seqLen ? GSFinishedByReachingSeqLen : GSInProgress);
      const int i = s.i;
      if (logprobsOut) (*logprobsOut)[(size_t)i].push_back(infContext.ReadLogprobs(seg_slot[j], curPos, 1)[0]);
      if (state != GSInProgress) { s.i = -1; live--; }
      emit(i, state, tok);
    }
  }
}
// EXTENSION: beam search (DESIGN.md §9f), the rules of the Python mirror's GenerateBeams.  NumBeams B in [1, 8]; a hypothesis
// of raw score s (the f64 sum of its tokens' logprobs) and n generated tokens ranks by h = s / pow(n, LengthPenalty).
struct BeamSearchArgs {
  int NumBeams = 1;
  double LengthPenalty = 1.0;
  bool EarlyStopping = false;
  int NumReturn = 1;
};
struct BeamHypothesis {
  std::vector<int32_t> Tokens;
  double Score = 0.0, NormalizedScore = 0.0;
  std::vector<double> Logprobs;
  GenerationState State = GSInProgress;
};

namespace beam_detail {
// -1: a before b, 1: after, 0: tie -- score descending, -inf after every finite score, NaN last
inline int ScoreOrder(double a, double b) {
  const bool na = std::isnan(a), nb = std::isnan(b);
  if (na || nb) return (int)na - (int)nb;
  return a > b ? -1 : a < b ? 1 : 0;
}
struct Cand { double score, lp; int beam, rank; int32_t token; };
// the pool: the best B by h, ties won by the earlier insertion
struct Pool {
  int B;
  std::vector<std::pair<BeamHypothesis, int64_t>> items;
  int64_t n_ins = 0;
  static bool Worse(const std::pair<BeamHypothesis, int64_t>& a, const std::pair<BeamHypothesis, int64_t>& b) {
    const int c = ScoreOrder(a.first.NormalizedScore, b.first.NormalizedScore);
    return c ? c > 0 : a.second > b.second;
  }
  size_t WorstIndex() const {
    size_t w = 0;
    for (size_t j = 1; j < items.size(); j++)
      if (Worse(items[j], items[w])) w = j;
    return w;
  }
  void Add(BeamHypothesis h) {
    const int64_t ins = n_ins++;
    if ((int)items.size() < B) { items.emplace_back(std::move(h), ins); return; }
    const size_t w = WorstIndex();
    if (ScoreOrder(h.NormalizedScore, items[w].first.NormalizedScore) < 0) items[w] = {std::move(h), ins};
  }
  std::vector<BeamHypothesis> Result() const {
    auto v = items;
    std::sort(v.begin(), v.end(), [](const auto& a, const auto& b) { return Worse(b, a); });
    std::vector<BeamHypothesis> out;
    for (auto& e : v) out.push_back(e.first);
    return out;
  }
};
}  // namespace beam_detail

// The prompt is prefilled on sequence 0 and forked to the other beams (CopySequences); every step is one ForwardBatch of the B
// beams, whose logprob records (top 2B) give the candidates, then one CopySequences moves each surviving beam's parent rows.
// Returns the NumReturn best hypotheses, best first.  Beam search ranks the raw distribution deterministically: sampling,
// penalties, a grammar or speculation are an error.
inline std::vector<BeamHypothesis> GenerateBeams(model::LlamaTransformer& transformer, const model::Vocabulary& vocab, int sequenceLength,
                                                 int accMode, const std::vector<int32_t>& promptTokens, const BeamSearchArgs& beams,
                                                 const model::SamplingArgs* sampling = nullptr, const model::PenaltyArgs* penalties = nullptr,
                                                 const model::SpeculativeArgs* speculative = nullptr,
                                                 const model::Grammar* grammar = nullptr) {
  using beam_detail::Cand;
  if ((sampling && sampling->Samples()) || penalties || speculative || grammar)
    throw Error("beam search ranks the raw distribution deterministically: it takes no sampling, penalties, grammar or "
                "speculative decoding");
  const int B = beams.NumBeams;
  if (B < 1 || B > 8) throw Error("NumBeams " + std::to_string(B) + " must be in [1, 8]");
  if (!std::isfinite(beams.LengthPenalty)) throw Error("LengthPenalty must be finite");
  if (beams.NumReturn < 1 || beams.NumReturn > B) throw Error("NumReturn must be in [1, NumBeams]");
  const int L = (int)promptTokens.size();
  model::InferenceContext infContext(transformer, sequenceLength, accMode, std::max(8, L), B);
  const int seqLen = infContext.SequenceLength;
  if (L < 1 || L >= seqLen)
    throw Error("context SequenceLength " + std::to_string(seqLen) + " must be higher than prompt tokens length " + std::to_string(L));
  for (int b = 0; b < B; b++) infContext.SetLogprobs(b, 2 * B);
  const double alpha = beams.LengthPenalty;
  auto norm = [&](double s, size_t n) { return s / std::pow((double)n, alpha); };
  auto is_stop = [&](int32_t t) { return std::find(vocab.StopTokenIds.begin(), vocab.StopTokenIds.end(), t) != vocab.StopTokenIds.end(); };
  beam_detail::Pool pool{B, {}, 0};
  struct Live { std::vector<int32_t> g; double s; std::vector<double> lps; };
  std::vector<Live> live{{{}, 0.0, {}}};
  for (int k = 0; k < seqLen - L; k++) {
    if (k == 0) {
      infContext.ForwardArgmax(promptTokens, 0);
    } else {
      std::vector<int32_t> toks, pos((size_t)live.size(), L + k - 1);
      for (const Live& b : live) toks.push_back(b.g.back());
      infContext.ForwardBatch(toks, pos);
    }
    std::vector<Cand> cands;
    for (size_t b = 0; b < live.size(); b++) {
      const lnb_logprob r = infContext.ReadLogprobs((int)b, L + k, 1)[0];
      for (int j = 0; j < r.n_top; j++) cands.push_back({live[b].s + r.top_logprob[j], r.top_logprob[j], (int)b, j, r.top_token[j]});
    }
    std::sort(cands.begin(), cands.end(), [](const Cand& a, const Cand& b) {
      const int c = beam_detail::ScoreOrder(a.score, b.score);
      if (c) return c < 0;
      return a.beam != b.beam ? a.beam < b.beam : a.rank < b.rank;
    });
    std::vector<Cand> next;
    for (size_t i = 0; i < cands.size() && (int)next.size() < B; i++) {
      const Cand& c = cands[i];
      if (!is_stop(c.token)) { next.push_back(c); continue; }
      if ((int)i >= B) continue;
      BeamHypothesis h{live[(size_t)c.beam].g, c.score, 0.0, live[(size_t)c.beam].lps, GSFinishedByReachingEOS};
      h.Tokens.push_back(c.token);
      h.Logprobs.push_back(c.lp);
      h.NormalizedScore = norm(c.score, h.Tokens.size());
      pool.Add(std::move(h));
    }
    if ((int)next.size() < B) break;   // fewer than B new beams: the search ends with the pool it has
    std::vector<Live> nl;
    std::vector<int32_t> parent;
    for (const Cand& c : next) {
      Live b = live[(size_t)c.beam];
      b.g.push_back(c.token);
      b.lps.push_back(c.lp);
      b.s = c.score;
      nl.push_back(std::move(b));
      parent.push_back(c.beam);
    }
    live = std::move(nl);
    if (L + k == seqLen - 1) {   // the new tokens sit at the last position: every live beam finishes, in beam order
      for (const Live& b : live) pool.Add(BeamHypothesis{b.g, b.s, norm(b.s, b.g.size()), b.lps, GSFinishedByReachingSeqLen});
      break;
    }
    if ((int)pool.items.size() == B) {
      double best = norm(live[0].s, live[0].g.size());
      for (const Live& b : live)
        if (beam_detail::ScoreOrder(norm(b.s, b.g.size()), best) < 0) best = norm(b.s, b.g.size());
      if (beams.EarlyStopping || beam_detail::ScoreOrder(best, pool.items[pool.WorstIndex()].first.NormalizedScore) >= 0) break;
    }
    std::vector<int32_t> src, dst;
    for (int i = 0; i < B; i++)
      if (parent[(size_t)i] != i) { src.push_back(parent[(size_t)i]); dst.push_back(i); }
    if (!src.empty()) infContext.CopySequences(src, dst, k == 0 ? 0 : L, L + k);   // the prompt after the prefill, later the generated rows
  }
  std::vector<BeamHypothesis> out = pool.Result();
  if ((int)out.size() > beams.NumReturn) out.resize((size_t)beams.NumReturn);
  return out;
}
}  // namespace inference
}  // namespace lnb_host
