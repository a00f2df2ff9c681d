// lnb_generate -- the cmd/main.go of this repository for the synthetic checkpoint: loads (random-inits)
// Llama-3.1-8B on device 0 through the C++ host mirror, runs the reference generate loop on the fixed
// 8-token prompt and prints the generated token ids and the decode rate.
// Build: make -C host      Run: host/lnb_generate [seq_len=136] [strict|fast] [tiny | <modelDir>] [batch=N] [logprobs=N]
// batch=N: N prompts (SURVEY 8d: prompt b = ids[1:] + 977 b) generated together, one pass over the weights per step.
// batch=N slots=K: the same N prompts through K live sequences with continuous batching (inference::GenerateTokensContinuous).
// temp=T [top_k=K] [top_p=P] [seed=S]: seeded sampling instead of the greedy argmax (lnb_session_set_sampling); prompt b of a
// batch samples with seed S + b.
// spec=K: speculative decoding -- each call verifies the last token plus up to K prompt-lookup drafts in one pass over the
// weights (lnb_forward_speculative); the generated ids are the same as without it.  Not with slots=.  branches=B (with spec=K):
// each call verifies a tree of up to K prompt-lookup nodes holding the top B continuations (lnb_forward_speculative_tree).
// rep=R freq=F pres=P [last_n=N]: repetition, frequency and presence penalties over the generated tokens (the last N positions;
// 0, the default: all) before the sampler or the greedy pick (lnb_session_set_penalties).
// regex=PATTERN (with <modelDir>/tokenizer.model): every generated token keeps the text a prefix of a string of
// re.fullmatch(PATTERN, s, re.ASCII); a stop token of the tokenizer only follows a complete match (model::Grammar,
// lnb_session_set_grammar).  Also with batch= (every prompt) and slots=; not with beams=.
// beams=B [len_pen=A] [early_stop=1]: beam search with B in [1, 8] beams (inference::GenerateBeams): one line per hypothesis,
// best first, with its state (1 EOS, 2 SequenceLength), raw score s and normalised score h = s / len^A, then its tokens (or
// text with a tokenizer).  Not with batch=, temp=, spec= or the penalties.
// logprobs=N (0..20): after the generated ids, one line per generated token with its logprob, its rank and the top N
// alternatives (lnb_session_set_logprobs; the raw model distribution, also for sampled tokens).
// score=TEXT (with <modelDir>/tokenizer.model): TEXT is tokenized without the chat template and scored in chunks of 64 tokens
// (lnb_score): each token's logprob given the tokens before it, their sum and the perplexity exp(-mean).
// prompt=TEXT (with <modelDir>/tokenizer.model): TEXT goes through the chat template and the BPE tokenizer, the
// generated ids come back as text (cmd/main.go's flow without the console UI).
// weights=mxfp8: the linear weights are quantized to MXFP8 at load (DESIGN §9h): half the weight bytes per step, and the
// same ids as the bf16 model whose weights are the dequantized values.  weights=mxfp4: the same with 4-bit codes (DESIGN §9i).
// <modelDir> holds params.json + consolidated.00.pth (model.LoadModel, src/model/loader.go:18-70);
// `lnb_generate --write-synthetic <modelDir> [tiny]` writes such a directory for the synthetic weights (host-only).
// `lnb_generate --tokenize <tokenizer.model> <text>` prints the chat-template token ids of <text> (host-only).
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "lnb_host.hpp"

using namespace lnb_host;

static void print_logprob(const char* tag, const lnb_logprob& r) {
  printf("%s %d %d %.17g |", tag, r.token, r.rank, r.logprob);
  for (int j = 0; j < r.n_top; j++) printf(" %d:%.17g", r.top_token[j], r.top_logprob[j]);
  printf("\n");
}

// score=TEXT: chunks of kScoreRows scored rows, each call overlapping the previous one by a token
static const int kScoreRows = 64;
static void score_text(model::LlamaTransformer& transformer, const model::Tokenizer& tok, int seq_len, int acc, const char* text) {
  const std::vector<int32_t> ids = tok.TokenizeString(text);
  const int n = (int)ids.size();
  if (n < 2) throw Error("score= needs a text of at least two tokens");
  if (n - 1 > seq_len) throw Error("score= text of " + std::to_string(n) + " tokens exceeds SequenceLength " + std::to_string(seq_len) + " + 1");
  model::InferenceContext ctx(transformer, seq_len, acc, kScoreRows);
  ctx.AllowChunkedPrefill(true);
  ctx.SetLogprobs(0, 0);
  std::vector<lnb_logprob> recs;
  for (int start = 0; start + 1 < n; start += kScoreRows) {
    const int end = std::min(n, start + kScoreRows + 1);
    const std::vector<lnb_logprob> r = ctx.Score(std::vector<int32_t>(ids.begin() + start, ids.begin() + end), start);
    recs.insert(recs.end(), r.begin(), r.end());
  }
  double sum = 0.0;
  for (size_t i = 0; i < recs.size(); i++) {
    printf("score %zu %d %.17g\n", i + 1, recs[i].token, recs[i].logprob);
    sum += recs[i].logprob;
  }
  printf("sum %.17g\nperplexity %.17g\n", sum, std::exp(-sum / (double)recs.size()));
}

static int write_synthetic_dir(const char* dir, bool tiny) {
  model::ModelArgs args = model::ModelArgs::Llama31_8B();
  const char* params = "{\"dim\": 4096, \"n_layers\": 32, \"n_heads\": 32, \"n_kv_heads\": 8, \"vocab_size\": 128256, "
                       "\"ffn_dim_multiplier\": 1.3, \"multiple_of\": 1024, \"norm_eps\": 1e-05, \"rope_theta\": 500000.0, "
                       "\"use_scaled_rope\": true}\n";
  if (tiny) {
    args.dim = 256; args.n_layers = 2; args.n_heads = 8; args.n_kv_heads = 2; args.head_dim = 32; args.ffn_dim = 512;
    args.vocab_size = 1024; args.max_seq_len = 64;
    params = "{\"dim\": 256, \"n_layers\": 2, \"n_heads\": 8, \"n_kv_heads\": 2, \"vocab_size\": 1024, \"ffn_dim_multiplier\": 0.75, "
             "\"multiple_of\": 256, \"norm_eps\": 1e-05, \"rope_theta\": 500000.0, \"use_scaled_rope\": true}\n";
  }
  const std::string d(dir);
  FILE* f = fopen((d + "/params.json").c_str(), "w");
  if (!f) { fprintf(stderr, "error: cannot write %s/params.json\n", dir); return 1; }
  fputs(params, f);
  fclose(f);
  check(lnb_pth_write_synthetic((d + "/consolidated.00.pth").c_str(), &args, tiny ? 7 : 0x4C4E42));
  check(lnb_vocab_write_synthetic((d + "/tokenizer.model").c_str(), args.vocab_size - 256));   // + 256 special tokens
  printf("wrote %s/params.json, %s/consolidated.00.pth and %s/tokenizer.model\n", dir, dir, dir);
  return 0;
}

int main(int argc, char** argv) {
  if (argc > 2 && !strcmp(argv[1], "--write-synthetic")) {
    try {
      return write_synthetic_dir(argv[2], argc > 3 && !strcmp(argv[3], "tiny"));
    } catch (const std::exception& e) {
      fprintf(stderr, "error: %s\n", e.what());
      return 1;
    }
  }
  if (argc > 3 && !strcmp(argv[1], "--tokenize")) {   // host-only: chat template + BPE + round trip
    try {
      model::Tokenizer tok(argv[2]);
      const std::vector<int32_t> ids = tok.Tokenize({{"user", argv[3]}});
      printf("ids:");
      for (int32_t t : ids) printf(" %d", t);
      printf("\ntext: %s\n", tok.TokenBatchToString(ids).c_str());
      return 0;
    } catch (const std::exception& e) {
      fprintf(stderr, "error: %s\n", e.what());
      return 1;
    }
  }
  if (argc > 3 && !strcmp(argv[1], "--detok-stream")) {   // host-only: streaming TokenToString over the given ids
    try {
      model::Tokenizer tok(argv[2]);
      std::string waiting, text;
      for (int i = 3; i < argc; i++) {
        const bool added = tok.TokenToString(atoi(argv[i]), waiting, text);
        printf("%d %s [%s]\n", atoi(argv[i]), added ? "waiting" : "text", text.c_str());
      }
      return 0;
    } catch (const std::exception& e) {
      fprintf(stderr, "error: %s\n", e.what());
      return 1;
    }
  }
  const int seq_len = argc > 1 ? atoi(argv[1]) : 136;
  const int acc = (argc > 2 && !strcmp(argv[2], "fast")) ? LNB_ACC_FAST : LNB_ACC_STRICT;
  const bool tiny = argc > 3 && !strcmp(argv[3], "tiny");
  const bool has_dir = argc > 3 && !tiny && strncmp(argv[3], "batch=", 6) != 0 && strncmp(argv[3], "weights=", 8) != 0;
  try {
    model::ModelArgs args = model::ModelArgs::Llama31_8B();
    std::vector<int32_t> prompt{128000, 9906, 11, 856, 836, 374, 220, 16};
    if (tiny) {
      args.dim = 256; args.n_layers = 2; args.n_heads = 8; args.n_kv_heads = 2; args.head_dim = 32; args.ffn_dim = 512;
      args.vocab_size = 1024; args.max_seq_len = 64;
      prompt = {1, 50, 999, 7, 300, 12, 64, 2};
    }
    const bool from_dir = has_dir;
    int weight_format = LNB_WEIGHTS_BF16;
    for (int i = 3; i < argc; i++) {
      if (!strcmp(argv[i], "weights=mxfp8")) weight_format = LNB_WEIGHTS_MXFP8;
      else if (!strcmp(argv[i], "weights=mxfp4")) weight_format = LNB_WEIGHTS_MXFP4;
      else if (!strncmp(argv[i], "weights=", 8) && strcmp(argv[i], "weights=bf16")) throw lnb_host::Error(std::string("unknown ") + argv[i]);
    }
    std::unique_ptr<model::LlamaTransformer> loaded;
    if (from_dir) {
      loaded = model::LoadModel(argv[3], 0, 2048, weight_format);
      if (loaded->args.vocab_size < 128256) prompt = {1, 50, 999, 7, 300, 12, 64, 2};
    } else {
      loaded = std::make_unique<model::LlamaTransformer>(args, 0);
      loaded->SetWeightFormat(weight_format);
      loaded->InitSynthetic(tiny ? 7 : 0x4C4E42);
      loaded->Finalize();
    }
    model::LlamaTransformer& transformer = *loaded;
    model::Vocabulary vocab;
    if (tiny || transformer.args.vocab_size < 128256) vocab.StopTokenIds = {1000000000};
    int batch = 0, slots = 0;
    const char* prompt_text = nullptr;
    const char* score_text_arg = nullptr;
    const char* regex = nullptr;
    int logprobs = -1;              // logprobs=N: top N alternatives per generated token
    model::SamplingArgs sampling;   // temp= top_k= top_p= seed= (temp 0, the default: greedy)
    model::SpeculativeArgs spec;    // spec=K: speculative decoding with up to K prompt-lookup drafts per call (0: plain steps)
    model::PenaltyArgs pen;         // rep= freq= pres= last_n= (the defaults: off)
    inference::BeamSearchArgs beam_args;   // beams= len_pen= early_stop= (NumBeams 0: no beam search)
    beam_args.NumBeams = 0;
    for (int i = 1; i < argc; i++) {
      if (!strncmp(argv[i], "rep=", 4)) pen.RepetitionPenalty = (float)atof(argv[i] + 4);
      if (!strncmp(argv[i], "freq=", 5)) pen.FrequencyPenalty = (float)atof(argv[i] + 5);
      if (!strncmp(argv[i], "pres=", 5)) pen.PresencePenalty = (float)atof(argv[i] + 5);
      if (!strncmp(argv[i], "last_n=", 7)) pen.Window = atoi(argv[i] + 7);
      if (!strncmp(argv[i], "beams=", 6)) beam_args.NumBeams = atoi(argv[i] + 6);
      if (!strncmp(argv[i], "len_pen=", 8)) beam_args.LengthPenalty = atof(argv[i] + 8);
      if (!strncmp(argv[i], "early_stop=", 11)) beam_args.EarlyStopping = atoi(argv[i] + 11) != 0;
      if (!strncmp(argv[i], "spec=", 5)) spec.MaxDraft = atoi(argv[i] + 5);
      if (!strncmp(argv[i], "branches=", 9)) spec.Branches = atoi(argv[i] + 9);
      if (!strncmp(argv[i], "batch=", 6)) batch = atoi(argv[i] + 6);
      if (!strncmp(argv[i], "slots=", 6)) slots = atoi(argv[i] + 6);
      if (!strncmp(argv[i], "prompt=", 7)) prompt_text = argv[i] + 7;
      if (!strncmp(argv[i], "score=", 6)) score_text_arg = argv[i] + 6;
      if (!strncmp(argv[i], "regex=", 6)) regex = argv[i] + 6;
      if (!strncmp(argv[i], "logprobs=", 9)) logprobs = atoi(argv[i] + 9);
      if (!strncmp(argv[i], "temp=", 5)) sampling.Temperature = (float)atof(argv[i] + 5);
      if (!strncmp(argv[i], "top_k=", 6)) sampling.TopK = atoi(argv[i] + 6);
      if (!strncmp(argv[i], "top_p=", 6)) sampling.TopP = (float)atof(argv[i] + 6);
      if (!strncmp(argv[i], "seed=", 5)) sampling.Seed = strtoull(argv[i] + 5, nullptr, 10);
    }
    std::unique_ptr<model::Tokenizer> tokenizer;
    if (score_text_arg) {
      if (!from_dir) throw Error("score= needs a model directory with tokenizer.model");
      score_text(transformer, model::Tokenizer(std::string(argv[3]) + "/tokenizer.model"), seq_len, acc, score_text_arg);
      return 0;
    }
    if (prompt_text || regex) {
      if (!from_dir) throw Error(std::string(prompt_text ? "prompt=" : "regex=") + " needs a model directory with tokenizer.model");
      tokenizer = std::make_unique<model::Tokenizer>(std::string(argv[3]) + "/tokenizer.model");
      if (tokenizer->Size() != transformer.args.vocab_size)   // checkModelArgs (loader.go:98-120)
        throw Error("VocabSize=" + std::to_string(transformer.args.vocab_size) + " and vocabulary model length=" +
                    std::to_string(tokenizer->Size()) + " aren't equal");
      vocab = tokenizer->GetVocabulary();
      if (prompt_text) prompt = tokenizer->Tokenize({{"user", prompt_text}});
    }
    std::unique_ptr<model::Grammar> grammar_owned;
    if (regex) grammar_owned = std::make_unique<model::Grammar>(transformer, regex, *tokenizer);
    const model::Grammar* grammar = grammar_owned.get();
    const model::SpeculativeArgs* speculative = spec.MaxDraft > 0 ? &spec : nullptr;
    const model::PenaltyArgs* penalties = pen.Neutral() ? nullptr : &pen;
    if (speculative && slots > 0) throw Error("spec= is not built for continuous batching (slots=)");
    if (beam_args.NumBeams != 0) {
      if (batch > 0) throw Error("beams= is not built with batch=");
      beam_args.NumReturn = std::max(1, beam_args.NumBeams);
      const std::vector<inference::BeamHypothesis> hyps =
          inference::GenerateBeams(transformer, vocab, seq_len, acc, prompt, beam_args, &sampling, penalties, speculative, grammar);
      for (size_t i = 0; i < hyps.size(); i++) {
        const inference::BeamHypothesis& h = hyps[i];
        printf("beam[%zu]: state %d s %.17g h %.17g |", i, (int)h.State, h.Score, h.NormalizedScore);
        if (tokenizer) printf(" text: %s", tokenizer->TokenBatchToString(h.Tokens).c_str());
        else
          for (int32_t t : h.Tokens) printf(" %d", t);
        printf("\n");
      }
      return 0;
    }
    if (batch > 0) {
      const int mod = transformer.args.vocab_size < 128256 ? 1000 : 128000;
      std::vector<std::vector<int32_t>> prompts(batch, prompt);
      for (int b = 0; b < batch; b++)
        for (size_t j = 1; j < prompt.size(); j++) prompts[b][j] = (prompt[j] + 977 * b) % mod;
      std::vector<std::vector<int32_t>> outs(batch);
      std::vector<std::vector<lnb_logprob>> lps;
      auto b0 = std::chrono::steady_clock::now();
      auto collect = [&](int seq, inference::GenerationState, int32_t tok) { outs[seq].push_back(tok); };
      if (slots > 0)
        inference::GenerateTokensContinuous(transformer, vocab, seq_len, acc, prompts, slots, std::max(slots, 64), collect, &sampling, logprobs,
                                            &lps, penalties, grammar);
      else
        inference::GenerateTokensBatch(transformer, vocab, seq_len, acc, prompts, collect, &sampling, speculative, logprobs, &lps, penalties,
                                       grammar);
      const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - b0).count();
      size_t total = 0;
      for (int b = 0; b < batch; b++) {
        printf("tokens[%d]:", b);
        for (int32_t t : outs[b]) printf(" %d", t);
        printf("\n");
        const std::string tag = "logprob[" + std::to_string(b) + "]:";
        if (logprobs >= 0)
          for (const lnb_logprob& r : lps[(size_t)b]) print_logprob(tag.c_str(), r);
        total += outs[b].size();
      }
      printf("generated %zu tokens for %d prompts in %.1f ms = %.1f tokens/s aggregate (prefill included)\n", total, batch, sec * 1e3, total / sec);
      return 0;
    }
    std::vector<int32_t> out;
    std::vector<lnb_logprob> lp;
    auto t0 = std::chrono::steady_clock::now();
    std::chrono::steady_clock::time_point t_first;
    inference::GenerateTokens(transformer, vocab, seq_len, acc, prompt, [&](inference::GenerationState, int32_t tok) {
      if (out.empty()) t_first = std::chrono::steady_clock::now();
      out.push_back(tok);
    }, &sampling, speculative, logprobs, &lp, penalties, grammar);
    auto t1 = std::chrono::steady_clock::now();
    if (tokenizer) printf("text: %s\n", tokenizer->TokenBatchToString(out).c_str());
    printf("tokens:");
    for (int32_t t : out) printf(" %d", t);
    const double dec_s = std::chrono::duration<double>(t1 - t_first).count();
    printf("\ngenerated %zu tokens (%s); prefill+first token %.1f ms; decode %.2f tokens/s through the reference-shaped host loop\n",
           out.size(), acc == LNB_ACC_STRICT ? "strict" : "fast", std::chrono::duration<double>(t_first - t0).count() * 1e3,
           out.size() > 1 ? (out.size() - 1) / dec_s : 0.0);
    for (const lnb_logprob& r : lp) print_logprob("logprob:", r);
  } catch (const std::exception& e) {
    fprintf(stderr, "error: %s\n", e.what());
    return 1;
  }
  return 0;
}
