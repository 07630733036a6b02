// The drop-in boundary: the reference's 17 `ctransformers_llm_*` C entry points
// (reference: models/llm.cc:32-138, bound by ctransformers/llm.py:117-208), re-implemented on top of the
// H100 engine, plus additive `ctb_*` entry points (declared in include/ctransformers_b200.h).
//
// Same semantics as the reference class LLM / llama_llm (models/llm.h:13-138, models/llms/llama.cc:10-117):
//   * create → nullptr (+ message on stderr) on any failure; nothing throws across the ABI
//   * batch_eval chunks by min(batch_size, n_ctx), clamps n_past to n_ctx - chunk (llm.h:40-54, 124-137)
//   * logits_data is a writable host pointer to the last token's n_vocab logits, valid until the next eval
//   * sample reseeds the RNG on every call (llama.cc:57-60)
// There is NO CPU fallback: without a CUDA device create fails loudly.
#include <algorithm>
#include <atomic>
#include <cctype>
#include <cmath>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "../../include/ctransformers_b200.h"
#include "beam.hpp"
#include "engine.cuh"
#include "gguf.hpp"
#include "grammar.hpp"
#include "sample_gpu.cuh"
#include "sampler.hpp"
#include "tp_nccl.hpp"
#include "vocab.hpp"

using namespace ctb;

static std::atomic<int> g_tp_ranks{0};   // live LLMs of the tensor-sharded mode in this process

struct LLM {
  ~LLM() {
    engine.reset();   // before the communicator its graphs captured
    if (comm) {
      NcclApi::get().CommDestroy((ncclComm_t)comm);
      g_tp_ranks--;
    }
  }
  void* comm = nullptr;   // ncclComm_t of the tensor-sharded mode
  std::unique_ptr<GGUFFile> file;
  Vocab vocab;
  HParams hp;
  std::unique_ptr<Engine> engine;
  std::string arch;
  std::string piece_buf;
  std::mt19937 rng;
  bool has_logits = false;
  long gpu_samples = 0;   // sample() calls answered by the device-side penalty + top-k
  long grammar_paths[3] = {0, 0, 0};   // constrained draws: device, host mask after a device bound, host cut (ctb_llm_grammar_paths)
  uint64_t fingerprint = 0;   // of the model file, computed on first use (model_fingerprint)
};

static bool file_is_gguf(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) return false;
  uint32_t magic = 0;
  const size_t n = fread(&magic, 1, 4, f);
  fclose(f);
  return n == 4 && magic == 0x46554747u;
}

static HParams read_hparams(const GGUFFile& g, const std::string& arch, int n_ctx_req) {
  HParams hp;
  hp.falcon = arch == "falcon";
  const GGUFValue* toks = g.find("tokenizer.ggml.tokens");
  if (!toks) throw std::runtime_error("key not found in model: tokenizer.ggml.tokens");
  hp.n_vocab = (int)toks->arr_n;
  hp.n_ctx_train = (int)g.need_u32(arch + ".context_length");
  hp.n_embd = (int)g.need_u32(arch + ".embedding_length");
  hp.n_ff = (int)g.need_u32(arch + ".feed_forward_length");
  hp.n_head = (int)g.need_u32(arch + ".attention.head_count");
  hp.n_layer = (int)g.need_u32(arch + ".block_count");
  hp.n_head_kv = (int)g.get_u32(arch + ".attention.head_count_kv", (uint32_t)hp.n_head);
  // reference llama.cpp:1576-1595: model values override the (default) context params
  hp.rope_base = g.get_f32(arch + ".rope.freq_base", 10000.0f);
  const float lin = g.get_f32(arch + ".rope.scale_linear", 1.0f);
  hp.rope_scale = lin != 1.0f ? 1.0f / lin : 1.0f;
  if (hp.n_head <= 0 || hp.n_embd % hp.n_head) throw std::runtime_error("invalid head count");
  hp.n_rot = (int)g.get_u32(arch + ".rope.dimension_count", (uint32_t)(hp.n_embd / hp.n_head));
  if (hp.n_rot != hp.n_embd / hp.n_head) throw std::runtime_error("invalid n_rot");
  hp.eps = hp.falcon ? g.need_f32(arch + ".attention.layer_norm_epsilon") : g.need_f32(arch + ".attention.layer_norm_rms_epsilon");
  hp.n_ctx = n_ctx_req > 0 ? n_ctx_req : 512;   // llama_context_default_params().n_ctx (llama.cpp:5281)
  if (hp.n_head_kv <= 0 || hp.n_head % hp.n_head_kv) throw std::runtime_error("invalid kv head count");
  const int hd = hp.head_dim();
  if (!attn_head_dim_ok(hd)) throw std::runtime_error("unsupported head size " + std::to_string(hd) + " (the CUDA path handles even sizes from 32 to 256)");
  return hp;
}

// LLM::BatchEval (llm.h:40-54): chunks of batch_size tokens, n_past clamped per chunk (llm.h:126).  The chunk a token belongs to
// fixes the row length n_total = n_past + N of its attention mat-muls.
static void eval_positions(int n_tokens, int n_past, int batch_size, int n_ctx, int* pos, int* nt) {
  const int bs = std::max(1, std::min(n_ctx, batch_size));
  int past = n_past;
  for (int start = 0; start < n_tokens; start += bs) {
    const int n = std::min(bs, n_tokens - start);
    const int p = std::max(0, std::min(n_ctx - n, past));
    for (int i = 0; i < n; i++) {
      pos[start + i] = p + i;
      nt[start + i] = p + n;
    }
    past += n;
  }
}

// The token list of one multi-sequence eval and its batched launches.  Slot slots[i] evaluates its tokens [off[i], off[i+1]) at
// n_past[i], with the positions and row lengths eval_positions gives that slot alone.  The lists are concatenated in call order
// and cut into launches of MULTI_LAUNCH_TOKENS (the batched kernel's PB_T), so a slot's token never runs in an earlier launch than the token before it.  A launch
// also ends where a slot's next position is not one past its previous one in the launch: a clamped chunk evaluates positions
// again, and their K / V may only be stored after the earlier tokens have read the old rows.  Returns the launch starts, the
// last entry being the token count.  tokens may be null (token ids 0).
static std::vector<int> multi_pack(int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size, int n_ctx,
                                   std::vector<MultiTok>& toks) {
  toks.clear();
  std::vector<int> starts(1, 0), pos, nt;
  for (int i = 0; i < n; i++) {
    const int m = off[i + 1] - off[i];
    if (m < 0) throw std::runtime_error("token offsets must not decrease");
    pos.resize(m); nt.resize(m);
    eval_positions(m, n_past[i], batch_size, n_ctx, pos.data(), nt.data());
    for (int j = 0; j < m; j++) {
      const int cur = (int)toks.size() - starts.back();
      const bool same_run = j > 0 && cur > 0 && pos[j] == pos[j - 1] + 1;
      if (cur == MULTI_LAUNCH_TOKENS || (j > 0 && cur > 0 && !same_run)) starts.push_back((int)toks.size());
      toks.push_back({slots[i], tokens ? tokens[off[i] + j] : 0, pos[j], nt[j], j == m - 1});
    }
  }
  if ((int)toks.size() > starts.back()) starts.push_back((int)toks.size());
  return starts;
}

// ---- sequence states (include/ctransformers_b200.h ctb_state_header)
static void fnv(uint64_t& h, const void* p, size_t n) {
  const uint8_t* b = (const uint8_t*)p;
  for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 0x100000001b3ull; }
}
static void fnv_str(uint64_t& h, const std::string& s) {
  const uint64_t n = s.size();
  fnv(h, &n, 8);
  fnv(h, s.data(), s.size());
}

// FNV-1a over the metadata, the tensor table and the first 4 KiB of every tensor's data: two files of the same shape differ in
// their weights, and reading every weight would cost as much as loading the model.
static uint64_t model_fingerprint(LLM& L) {
  if (L.fingerprint) return L.fingerprint;
  const GGUFFile& g = *L.file;
  uint64_t h = 0xcbf29ce484222325ull;
  fnv(h, &g.version, 4);
  for (const auto& [key, v] : g.kv) {
    fnv_str(h, key);
    fnv(h, &v.type, 4); fnv(h, &v.u, 8); fnv(h, &v.f, 8); fnv_str(h, v.s);
    fnv(h, &v.arr_type, 4); fnv(h, &v.arr_n, 8);
    if (v.arr_data) fnv(h, v.arr_data, GGUFFile::scalar_size(v.arr_type) * v.arr_n);
    for (const std::string& s : v.arr_str) fnv_str(h, s);
  }
  for (const GGUFTensor& t : g.tensors) {
    fnv_str(h, t.name);
    fnv(h, &t.n_dims, 4); fnv(h, t.ne, sizeof(t.ne)); fnv(h, &t.type, 4); fnv(h, &t.offset, 8);
    fnv(h, t.data, (size_t)std::min<uint64_t>(t.nbytes, 4096));
  }
  return L.fingerprint = h ? h : 1;
}

static ctb_state_header state_header(LLM& L, int n_tokens, bool results) {
  ctb_state_header s{};
  s.magic = CTB_STATE_MAGIC;
  s.version = CTB_STATE_VERSION;
  s.n_layer = L.hp.n_layer; s.n_head_kv = L.hp.n_head_kv; s.head_dim = L.hp.head_dim(); s.k_stride = L.engine->state_k_stride();
  s.n_embd = L.hp.n_embd; s.n_vocab = L.hp.n_vocab;
  s.n_tokens = n_tokens;
  s.has_results = results ? 1 : 0;
  s.fingerprint = model_fingerprint(L);
  return s;
}

static uint64_t state_size(const ctb_state_header& s) {
  const uint64_t n = (uint64_t)s.n_tokens, n_pad = (n + 255) & ~255ull, rows = (uint64_t)s.n_layer * s.n_head_kv;
  return sizeof(ctb_state_header) + 4 * n + rows * (n * s.k_stride + n_pad * s.head_dim) * 2 +
         (s.has_results ? ((uint64_t)s.n_vocab + s.n_embd) * 4 : 0);
}

// Why buf cannot be a state ("" when it can); s gets its header.  The bounds keep state_size within 64 bits.
static std::string state_check(const void* buf, size_t size, ctb_state_header& s) {
  if (!buf || size < sizeof(s)) return "a state has at least a " + std::to_string(sizeof(s)) + "-byte header; this one has " + std::to_string(size) + " bytes";
  memcpy(&s, buf, sizeof(s));
  if (s.magic != CTB_STATE_MAGIC) return "not a sequence state (bad magic)";
  if (s.version != CTB_STATE_VERSION) return "state version " + std::to_string(s.version) + " (this library reads version " + std::to_string(CTB_STATE_VERSION) + ")";
  auto in = [](int32_t v, int32_t lo, int32_t hi) { return v >= lo && v <= hi; };
  if (!in(s.n_layer, 1, 4096) || !in(s.n_head_kv, 1, 4096) || !in(s.head_dim, 1, 4096) || !in(s.k_stride, s.head_dim, 4096) ||
      !in(s.n_embd, 1, 1 << 24) || !in(s.n_vocab, 1, 1 << 24) || !in(s.n_tokens, 0, 1 << 24) || !in(s.has_results, 0, 1))
    return "the state's header is malformed";
  if (state_size(s) != size)
    return "the state's size (" + std::to_string(size) + " bytes) disagrees with its header (" + std::to_string(state_size(s)) + " bytes)";
  return "";
}

static size_t state_size_for(LLM& L, int n_tokens) {
  if (n_tokens < 0 || n_tokens > L.hp.n_ctx) return 0;
  return (size_t)state_size(state_header(L, n_tokens, n_tokens > 0));
}

static void save_state(LLM& L, int slot, const int* tokens, int n_tokens, bool results, void* buf, size_t cap) {
  if (n_tokens < 0 || n_tokens > L.hp.n_ctx)
    throw std::runtime_error(std::to_string(n_tokens) + " tokens: a state holds 0 .. " + std::to_string(L.hp.n_ctx) + " (the context length)");
  if (n_tokens > 0 && !tokens) throw std::runtime_error("no tokens");
  const ctb_state_header s = state_header(L, n_tokens, results && n_tokens > 0);
  const uint64_t need = state_size(s);
  if (!buf || cap < need) throw std::runtime_error("the state needs " + std::to_string(need) + " bytes; the buffer has " + std::to_string(cap));
  uint8_t* p = (uint8_t*)buf;
  memcpy(p, &s, sizeof(s));
  memcpy(p + sizeof(s), tokens, (size_t)n_tokens * 4);
  L.engine->state_save(slot, n_tokens, s.has_results, p + sizeof(s) + (size_t)n_tokens * 4);
}

// Checks everything before the first device copy: a refused state leaves the slot as it was.  Returns the header.
static ctb_state_header restore_state(LLM& L, int slot, const void* buf, size_t size) {
  ctb_state_header s;
  std::string why = state_check(buf, size, s);
  const ctb_state_header want = state_header(L, 0, false);
  if (why.empty() && (s.n_layer != want.n_layer || s.n_head_kv != want.n_head_kv || s.head_dim != want.head_dim || s.k_stride != want.k_stride ||
                      s.n_embd != want.n_embd || s.n_vocab != want.n_vocab))
    why = "the state is of a model of another shape";
  if (why.empty() && s.fingerprint != want.fingerprint) why = "the state is of another model file";
  if (why.empty() && s.n_tokens > L.hp.n_ctx)
    why = "the state holds " + std::to_string(s.n_tokens) + " positions; the context length is " + std::to_string(L.hp.n_ctx);
  const uint8_t* p = (const uint8_t*)buf + sizeof(s);
  int last = 0;
  for (int i = 0; why.empty() && i < s.n_tokens; i++) {
    memcpy(&last, p + (size_t)i * 4, 4);
    if (last < 0 || last >= L.hp.n_vocab) why = "the state holds a token id out of range";
  }
  if (!why.empty()) throw std::invalid_argument(why);
  L.engine->state_load(slot, s.n_tokens, s.has_results, p + (size_t)s.n_tokens * 4, last);
  return s;
}

static int state_error(const char* what, const std::exception& e) {
  fprintf(stderr, "ctransformers-b200: %s: %s\n", what, e.what());
  return -1;
}

// What every handle loads: the model file, its architecture, hyper-parameters and vocabulary.  The model type is checked before
// anything needs a device (a GGUF file: model_type "gguf" or the file's magic).  Returns the CUDA device count.
static int load_model(LLM& L, const char* model_path, const char* model_type, int context_length) {
  std::string type = model_type ? model_type : "";
  type.erase(std::remove_if(type.begin(), type.end(), [](const char c) { return !std::isalnum((unsigned char)c); }), type.end());
  if (!(type == "gguf" || file_is_gguf(model_path)))
    throw std::runtime_error("model type '" + std::string(model_type ? model_type : "") + "' is not supported by this build (GGUF llama / falcon only)");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw std::runtime_error("no CUDA device available; this library has no CPU fallback");
  L.file.reset(new GGUFFile(model_path));
  L.arch = L.file->need_str("general.architecture");
  if (L.arch != "llama" && L.arch != "falcon") throw std::runtime_error("unknown model architecture: '" + L.arch + "'");
  L.hp = read_hparams(*L.file, L.arch, context_length);
  L.vocab.load(*L.file);
  return ndev;
}

// Refuses a tensor-sharded LLM what that mode does not have: "the tensor-sharded mode " + why.
static void not_sharded(LLM* llm, const char* why) {
  if (llm->comm) throw std::invalid_argument(std::string("the tensor-sharded mode ") + why);
}

static void check_tokens(const int* tokens, int n, int n_vocab) {
  if (n > 0 && !tokens) throw std::invalid_argument("no tokens");
  for (int i = 0; i < n; i++)
    if (tokens[i] < 0 || tokens[i] >= n_vocab) throw std::invalid_argument("token id out of range");
}

// targets: -1 (no target) or a token id
static void check_targets(const int* targets, int n, int n_vocab) {
  if (n > 0 && !targets) throw std::invalid_argument("no targets");
  for (int i = 0; i < n; i++)
    if (targets[i] < -1 || targets[i] >= n_vocab)
      throw std::invalid_argument("target " + std::to_string(targets[i]) + " of token " + std::to_string(i) + " is out of range (-1 .. " + std::to_string(n_vocab - 1) + ")");
}

// The eval of an LLM, 0 or -1.  The engine gets the whole list at once so that prompt chunks can share batched launches.  With
// a sink it also keeps every token's row.  Everything is checked before the first launch, so a refusal leaves the handle as it was.
static int llm_eval(LLM* llm, const int* tokens, int n_tokens, int n_past, int batch_size, const RowSink* sink, const char* what) {
  try {
    if (sink) not_sharded(llm, "keeps no per-token rows");
    check_tokens(tokens, n_tokens, llm->hp.n_vocab);
    if (sink && sink->targets) check_targets(sink->targets, n_tokens, llm->hp.n_vocab);
    else if (sink && n_tokens > 0 && !sink->host) throw std::invalid_argument("no memory for the rows");
    if (n_tokens <= 0) return 0;
    std::vector<int> pos(n_tokens), nt(n_tokens);
    eval_positions(n_tokens, n_past, batch_size, llm->hp.n_ctx, pos.data(), nt.data());
    llm->engine->eval_list(tokens, pos.data(), nt.data(), n_tokens, sink);
    llm->has_logits = true;
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: %s failed: %s\n", what, e.what());
    return -1;
  } catch (...) { return -1; }
}

extern "C" {

static LLM* create_llm(const char* model_path, const char* model_type, const ctransformers_config config, int rank, int world, const void* unique_id) {
  try {
    std::unique_ptr<LLM> llm(new LLM);
    const int ndev = load_model(*llm, model_path, model_type, config.context_length);
    int device = 0;
    if (const char* env = getenv("CT_DEVICE")) device = atoi(env);
    else if (const char* lr = getenv("LOCAL_RANK")) device = atoi(lr) % ndev;
    TPShard tp;
    if (world > 1) {
      if (!attn_fast_hd(llm->hp.head_dim())) throw std::runtime_error("tensor parallel: head size " + std::to_string(llm->hp.head_dim()) + " (this mode takes 64 and 128)");
      if (!unique_id) throw std::runtime_error("tensor parallel: no communicator id");
      tp = tp_shard(llm->hp.n_embd, llm->hp.n_head, llm->hp.n_head_kv, llm->hp.n_ff, rank, world);
      if (cudaSetDevice(device) != cudaSuccess) throw std::runtime_error("cudaSetDevice failed");
      const NcclApi& nccl = NcclApi::get();
      ncclUniqueId id;
      memcpy(&id, unique_id, sizeof(id));
      ncclComm_t comm = nullptr;
      nccl.check(nccl.CommInitRank(&comm, world, id, rank), "communicator init");
      llm->comm = comm;
      g_tp_ranks++;
      tp.comm = comm;
    }
    llm->engine.reset(new Engine(*llm->file, llm->hp, device, tp));
    return llm.release();
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: failed to load model: %s\n", e.what());
    return nullptr;
  } catch (...) {
    fprintf(stderr, "ctransformers-b200: failed to load model\n");
    return nullptr;
  }
}

LLM* ctransformers_llm_create(const char* model_path, const char* model_type, const ctransformers_config config) {
  return create_llm(model_path, model_type, config, 0, 1, nullptr);
}

int ctb_tp_unique_id(void* out, int cap) {
  try {
    if (!out || cap < (int)sizeof(ncclUniqueId)) return -(int)sizeof(ncclUniqueId);
    const NcclApi& nccl = NcclApi::get();
    ncclUniqueId id;
    nccl.check(nccl.GetUniqueId(&id), "unique id");
    memcpy(out, &id, sizeof(id));
    return (int)sizeof(id);
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: %s\n", e.what());
    return 0;
  } catch (...) { return 0; }
}

LLM* ctb_llm_create_tp(const char* model_path, const char* model_type, const ctransformers_config config, int rank, int world, const void* unique_id) {
  if (world < 1 || rank < 0 || rank >= world) {
    fprintf(stderr, "ctransformers-b200: bad tensor-parallel rank %d of %d\n", rank, world);
    return nullptr;
  }
  return create_llm(model_path, model_type, config, rank, world, unique_id);
}

int ctb_tp_shard(int n_embd, int n_head, int n_head_kv, int n_ff, int rank, int world, int* out6) {
  try {
    const TPShard s = tp_shard(n_embd, n_head, n_head_kv, n_ff, rank, world);
    out6[0] = s.head0; out6[1] = s.head1; out6[2] = s.kv0; out6[3] = s.kv1; out6[4] = s.ff0; out6[5] = s.ff1;
    return 0;
  } catch (...) { return -1; }
}

void ctransformers_llm_delete(LLM* llm) { delete llm; }

int ctransformers_llm_tokenize(LLM* llm, const char* text, const bool add_bos_token, int* output) {
  try {
    const std::vector<int> t = llm->vocab.tokenize(text ? text : "", add_bos_token);
    std::copy(t.begin(), t.end(), output);
    return (int)t.size();
  } catch (...) { return 0; }
}

const char* ctransformers_llm_detokenize(LLM* llm, const int token) {
  try {
    llm->piece_buf = llm->vocab.piece(token);
  } catch (...) { llm->piece_buf.clear(); }   // nothing may cross the C ABI
  return llm->piece_buf.c_str();
}

bool ctransformers_llm_is_eos_token(LLM* llm, const int token) { return token == llm->vocab.eos; }
int ctransformers_llm_eos_token_id(LLM* llm) { return llm->vocab.eos; }
int ctransformers_llm_bos_token_id(LLM* llm) { return llm->vocab.bos; }
int ctransformers_llm_vocab_size(LLM* llm) { return llm->hp.n_vocab; }
int ctransformers_llm_context_length(LLM* llm) { return llm->hp.n_ctx; }
const char* ctransformers_llm_architecture(LLM* llm) { return llm->arch.c_str(); }

bool ctransformers_llm_batch_eval(LLM* llm, const int* tokens, const int n_tokens, const int n_past, const int batch_size, const int threads) {
  (void)threads;   // host thread count has no meaning on the GPU path
  return llm_eval(llm, tokens, n_tokens, n_past, batch_size, nullptr, "eval") == 0;
}

float* ctransformers_llm_logits_data(LLM* llm) { return llm->engine->logits(); }
int ctransformers_llm_logits_size(LLM* llm) { return llm->has_logits ? llm->hp.n_vocab : 0; }
const float* ctransformers_llm_embeddings_data(LLM* llm) { return llm->engine->embeddings(); }
int ctransformers_llm_embeddings_size(LLM* llm) { return llm->has_logits ? llm->hp.n_embd : 0; }

int ctransformers_llm_sample(LLM* llm, const int* last_tokens, const int n_last, const int top_k, const float top_p, const float temperature,
                             const float repetition_penalty, int seed) {
  try {
    if (seed < 0) seed = (int)time(nullptr);
    llm->rng.seed((unsigned)seed);
    if (llm->engine->lazy_logits()) {
      // nobody holds a host view of the logits.  The engine already holds the greedy pick of these logits (its look-ahead pick).
      Engine& e = *llm->engine;
      bool used_device = false;
      const int t = sample_lazy(
          llm->hp.n_vocab, last_tokens, n_last, top_k, top_p, temperature, repetition_penalty, llm->rng, used_device, [&] { return e.greedy_pick(); },
          [&](const int* last, int nl, float pen, int k, int* ids, float* lg) { return e.topk_candidates(last, nl, pen, k, ids, lg); },
          [&] { return e.logits_copy(); });
      if (used_device) llm->gpu_samples++;
      return t;
    }
    return sample_token(llm->engine->logits(), llm->hp.n_vocab, last_tokens, n_last, top_k, top_p, temperature, repetition_penalty, llm->rng);
  } catch (...) { return llm->vocab.eos; }
}

void ctransformers_llm_reset(LLM* llm) { (void)llm; /* reference clears only the generic logits_ vector, which GGUF models do not use (llm.h:106, llama.cc:47) */ }

// ----------------------------------------------------------------------------- additive entry points
int ctb_abi_version(void) { return 1; }

double ctb_llm_last_eval_ms(LLM* llm) { return llm->engine->stats.last_eval_ms; }
long ctb_llm_launches_per_token(LLM* llm) { return llm->engine->stats.launches; }
long ctb_llm_speculative_hits(LLM* llm) { return llm->engine->stats.spec_hits; }
unsigned long long ctb_llm_weight_bytes_per_token(LLM* llm) { return (unsigned long long)llm->engine->stats.weight_bytes_per_token; }
long ctb_llm_device_samples(LLM* llm) { return llm->gpu_samples; }
double ctb_llm_load_ms(LLM* llm) { return llm->engine->stats.load_ms; }
void ctb_llm_set_stream(LLM* llm, void* cuda_stream) { llm->engine->set_stream((cudaStream_t)cuda_stream); }

double ctb_llm_decode_greedy(LLM* llm, int first_token, int n_past, int n_steps, int* out_tokens) {
  try {
    const double ms = llm->engine->decode_greedy(first_token, n_past, n_steps, out_tokens);
    llm->has_logits = true;
    return ms;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: decode_greedy failed: %s\n", e.what());
    return -1.0;
  }
}

int ctb_llm_profile_step(LLM* llm, int token, int n_past, double* ms_by_kind, int* count_by_kind) {
  try {
    return llm->engine->profile_step(token, n_past, ms_by_kind, count_by_kind);
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: profile_step failed: %s\n", e.what());
    return -1;
  }
}

long ctb_llm_trace_step(LLM* llm, int token, int n_past, unsigned long long* out, long cap_words) {
  try {
    return llm->engine->trace_step(token, n_past, out, cap_words);
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: trace_step failed: %s\n", e.what());
    return 0;
  }
}

long ctb_llm_paths(LLM* llm, int* out, int cap) {
  try {
    return llm->engine->paths(out, cap);
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: paths failed: %s\n", e.what());
    return -100;
  }
}

int ctb_llm_step_cluster(LLM* llm) { return llm->engine->step_cluster(); }

double ctb_llm_time_matvec_only(LLM* llm, int reps, long* launches) { return ctb_llm_time_matvec_kinds(llm, reps, launches, 0); }

double ctb_llm_time_matvec_kinds(LLM* llm, int reps, long* launches, unsigned kind_mask) {
  try {
    return llm->engine->time_matvec_only(reps < 1 ? 1 : reps, launches, kind_mask);
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: time_matvec_only failed: %s\n", e.what());
    return -1.0;
  }
}

int ctb_state_info(const void* buf, size_t size, ctb_state_header* out) {
  ctb_state_header s;
  const std::string why = state_check(buf, size, s);
  if (!why.empty()) {
    fprintf(stderr, "ctransformers-b200: %s\n", why.c_str());
    return -1;
  }
  if (out) *out = s;
  return 0;
}

size_t ctb_llm_state_size(LLM* llm, int n_tokens) {
  try {
    not_sharded(llm, "has no sequence states");
    return state_size_for(*llm, n_tokens);
  } catch (...) { return 0; }
}

int ctb_llm_save_state(LLM* llm, const int* tokens, int n_tokens, void* buf, size_t cap) {
  try {
    not_sharded(llm, "has no sequence states");
    save_state(*llm, 0, tokens, n_tokens, llm->has_logits, buf, cap);
    return 0;
  } catch (const std::exception& e) { return state_error("cannot save the state", e); }
}

int ctb_llm_load_state(LLM* llm, const void* buf, size_t size) {
  try {
    not_sharded(llm, "has no sequence states");
    llm->has_logits = restore_state(*llm, 0, buf, size).has_results != 0;
    return 0;
  } catch (const std::exception& e) { return state_error("cannot load the state", e); }
}

// ---- rows of every token (the reference's logits_all) and their scores
int ctb_llm_batch_eval_rows(LLM* llm, const int* tokens, int n_tokens, int n_past, int batch_size, float* rows) {
  RowSink s;
  s.host = rows;
  return llm_eval(llm, tokens, n_tokens, n_past, batch_size, &s, "eval with rows");
}

int ctb_llm_batch_eval_scored(LLM* llm, const int* tokens, int n_tokens, int n_past, int batch_size, const int* targets, double* logprob, int* greedy) {
  RowSink s;
  s.targets = targets; s.logprob = logprob; s.greedy = greedy;
  if (n_tokens > 0 && (!logprob || !greedy)) {
    fprintf(stderr, "ctransformers-b200: scored eval failed: no memory for the scores\n");
    return -1;
  }
  return llm_eval(llm, tokens, n_tokens, n_past, batch_size, &s, "scored eval");
}

int ctb_llm_score_last(LLM* llm, int target, double* logprob, int* greedy) {
  try {
    not_sharded(llm, "keeps no per-token rows");
    if (!llm->has_logits) throw std::invalid_argument("nothing has been evaluated");
    check_targets(&target, 1, llm->hp.n_vocab);
    llm->engine->score_kept(target, logprob, greedy);
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: scoring the last logits failed: %s\n", e.what());
    return -1;
  } catch (...) { return -1; }
}

// ---- host-only logic (no GPU needed): tokenizer / detokenizer / sampler on their own
struct ctb_vocab { std::unique_ptr<GGUFFile> file; Vocab vocab; };

ctb_vocab* ctb_vocab_load(const char* gguf_path) {
  try {
    std::unique_ptr<ctb_vocab> v(new ctb_vocab);
    v->file.reset(new GGUFFile(gguf_path));
    v->vocab.load(*v->file);
    return v.release();
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: ctb_vocab_load failed: %s\n", e.what());
    return nullptr;
  }
}
void ctb_vocab_free(ctb_vocab* v) { delete v; }
int ctb_vocab_size(ctb_vocab* v) { return v->vocab.size(); }
int ctb_vocab_tokenize(ctb_vocab* v, const char* text, bool add_bos, int* out, int cap) {
  try {
    const std::vector<int> t = v->vocab.tokenize(text ? text : "", add_bos);
    if ((int)t.size() > cap) return -(int)t.size();
    std::copy(t.begin(), t.end(), out);
    return (int)t.size();
  } catch (...) { return 0; }
}
int ctb_vocab_piece(ctb_vocab* v, int token, char* buf, int cap) {
  const std::string s = v->vocab.piece(token);
  if ((int)s.size() > cap) return -(int)s.size();
  memcpy(buf, s.data(), s.size());
  return (int)s.size();
}
// ---- multi-sequence handle: S slots, each a single-sequence LLM of its own, evaluated together in batched launches
struct ctb_multi {
  std::unique_ptr<LLM> llm;   // file, vocabulary, hyper-parameters and the engine (its KV cache holds n_slots regions)
  int n_slots = 0;
  std::vector<std::vector<float>> logits, embd;   // host copies, fetched on request
  std::vector<char> has, fresh;                   // the slot has results / its host copies are current
  long device_samples = 0;                        // draws answered on the device (LLM::gpu_samples of every slot)
  double beam_stats[8] = {0};                     // the last beam search: ctb_multi_beam_stats
};

static bool multi_slot_ok(ctb_multi* m, int slot) {
  if (slot >= 0 && slot < m->n_slots) return true;
  fprintf(stderr, "ctransformers-b200: slot %d is out of range (the handle has %d)\n", slot, m->n_slots);
  return false;
}

static bool multi_fetch(ctb_multi* m, int slot) {
  if (!multi_slot_ok(m, slot) || !m->has[slot]) return false;
  if (!m->fresh[slot]) {
    m->llm->engine->multi_fetch(slot, m->logits[slot].data(), m->embd[slot].data());
    m->fresh[slot] = 1;
  }
  return true;
}

ctb_multi* ctb_multi_create(const char* model_path, const char* model_type, const ctransformers_config config, int n_slots) {
  try {
    if (n_slots < 1) throw std::runtime_error("n_slots must be at least 1");
    std::unique_ptr<ctb_multi> m(new ctb_multi);
    m->llm.reset(new LLM);
    LLM& L = *m->llm;
    load_model(L, model_path, model_type, config.context_length);
    if (g_tp_ranks > 0)
      throw std::runtime_error("multi-sequence decoding in the tensor-sharded mode is not supported by the CUDA path");
    L.hp.n_seq = n_slots;
    L.hp.multi = true;
    for (const auto& t : L.file->tensors)
      if (t.n_dims >= 2 && t.name.rfind("blk.", 0) == 0 && !type_is_kquant((int)t.type))
        throw std::runtime_error("multi-sequence decoding of layer matrices that are not K-quants (tensor '" + t.name + "', type " + std::to_string(t.type) +
                                 ") is not supported by the CUDA path");
    int device = 0;
    if (const char* env = getenv("CT_DEVICE")) device = atoi(env);
    if (cudaSetDevice(device) != cudaSuccess) throw std::runtime_error("cudaSetDevice failed");
    size_t free_b = 0, total_b = 0;
    const size_t need = engine_arena_bytes(*L.file, L.hp);
    if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && need > free_b)
      throw std::runtime_error(std::to_string(n_slots) + " sequence slots need " + std::to_string(need) + " bytes of device memory; " + std::to_string(free_b) + " are free");
    L.engine.reset(new Engine(*L.file, L.hp, device));
    const std::string why = L.engine->multi_refusal();
    if (!why.empty()) throw std::runtime_error("multi-sequence decoding of " + why + " is not supported by the CUDA path");
    m->n_slots = n_slots;
    m->logits.assign(n_slots, std::vector<float>(L.hp.n_vocab));
    m->embd.assign(n_slots, std::vector<float>(L.hp.n_embd));
    m->has.assign(n_slots, 0);
    m->fresh.assign(n_slots, 0);
    return m.release();
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: failed to create the multi-sequence handle: %s\n", e.what());
    return nullptr;
  } catch (...) {
    fprintf(stderr, "ctransformers-b200: failed to create the multi-sequence handle\n");
    return nullptr;
  }
}

void ctb_multi_delete(ctb_multi* m) { delete m; }

int ctb_multi_info(ctb_multi* m, int* out6) {
  const HParams& hp = m->llm->hp;
  const int v[6] = {m->n_slots, hp.n_vocab, hp.n_embd, hp.n_ctx, m->llm->vocab.eos, m->llm->vocab.bos};
  std::copy(v, v + 6, out6);
  return 6;
}

// slots[0 .. n) are in range (false, with a message, when one is not) and listed once (else it throws)
static bool multi_slots_ok(ctb_multi* m, int n, const int* slots) {
  std::vector<char> seen(m->n_slots, 0);
  for (int i = 0; i < n; i++) {
    if (!multi_slot_ok(m, slots[i])) return false;
    if (seen[slots[i]]++) throw std::invalid_argument("slot " + std::to_string(slots[i]) + " is listed twice");
  }
  return true;
}

// The eval of a multi-sequence handle, 0 or -1; with a sink it also keeps the row of every token of the packed list (call order).
// Everything is checked before the first launch.
static int multi_eval(ctb_multi* m, int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size, const RowSink* sink,
                      const char* what) {
  try {
    if (!multi_slots_ok(m, n, slots)) return -1;
    const int total = n > 0 ? off[n] - off[0] : 0;
    check_tokens(tokens ? tokens + (n > 0 ? off[0] : 0) : nullptr, total, m->llm->hp.n_vocab);
    if (sink && sink->targets) check_targets(sink->targets, total, m->llm->hp.n_vocab);
    else if (sink && total > 0 && !sink->host) throw std::invalid_argument("no memory for the rows");
    std::vector<MultiTok> toks;
    const std::vector<int> starts = multi_pack(n, slots, off, tokens, n_past, batch_size, m->llm->hp.n_ctx, toks);
    if (toks.empty()) return 0;
    for (int i = 0; i < n; i++) m->fresh[slots[i]] = 0;
    m->llm->engine->multi_eval(toks, starts, sink);
    for (int i = 0; i < n; i++)
      if (off[i + 1] > off[i]) m->has[slots[i]] = 1;
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: %s failed: %s\n", what, e.what());
    return -1;
  } catch (...) { return -1; }
}

bool ctb_multi_eval(ctb_multi* m, int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size) {
  return multi_eval(m, n, slots, off, tokens, n_past, batch_size, nullptr, "multi-sequence eval") == 0;
}

int ctb_multi_eval_rows(ctb_multi* m, int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size, float* rows) {
  RowSink s;
  s.host = rows;
  return multi_eval(m, n, slots, off, tokens, n_past, batch_size, &s, "multi-sequence eval with rows");
}

int ctb_multi_eval_scored(ctb_multi* m, int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size, const int* targets,
                          double* logprob, int* greedy) {
  RowSink s;
  s.targets = targets; s.logprob = logprob; s.greedy = greedy;
  if (n > 0 && off[n] > off[0] && (!logprob || !greedy)) {
    fprintf(stderr, "ctransformers-b200: multi-sequence scored eval failed: no memory for the scores\n");
    return -1;
  }
  return multi_eval(m, n, slots, off, tokens, n_past, batch_size, &s, "multi-sequence scored eval");
}

const float* ctb_multi_logits(ctb_multi* m, int slot) {
  try { return multi_fetch(m, slot) ? m->logits[slot].data() : nullptr; } catch (...) { return nullptr; }
}
const float* ctb_multi_embeddings(ctb_multi* m, int slot) {
  try { return multi_fetch(m, slot) ? m->embd[slot].data() : nullptr; } catch (...) { return nullptr; }
}

// ctransformers_llm_sample on each listed slot, its draws in list order: slot slots[i] with the window last_tokens[last_off[i] ..
// last_off[i + 1]) and the i-th settings.  Everything is checked before the first draw; then every slot goes through
// sample_lazy, the chain an LLM runs on logits that are still on the device.  Its device half runs for all slots at once
// (Engine::multi_sample): one k_sample_topk launch over the slots that need a cut and that the kernel takes, one copy back of
// those results and of every slot's greedy pick.  Greedy slots need no cut: their pick answers, and where it cannot (equal
// maxima, NaN) a cut of 1 cannot either.  What the device cannot answer goes to the host sampler on that slot's logits.
int ctb_multi_sample_many(ctb_multi* m, int n, const int* slots, const int* last_off, const int* last_tokens, const int* top_k, const float* top_p,
                          const float* temperature, const float* repetition_penalty, const int* seed, int* out) {
  try {
    if (n < 0) throw std::invalid_argument("a negative slot count");
    if (n > 0 && (!slots || !last_off || !top_k || !top_p || !temperature || !repetition_penalty || !seed || !out))
      throw std::invalid_argument("a missing argument array");
    if (!multi_slots_ok(m, n, slots)) return -1;
    for (int i = 0; i < n; i++) {
      if (!m->has[slots[i]]) throw std::invalid_argument("slot " + std::to_string(slots[i]) + " has no logits to sample from");
      if (last_off[i] < 0 || last_off[i + 1] < last_off[i]) throw std::invalid_argument("the window offsets of slot " + std::to_string(slots[i]) + " are not ascending");
    }
    if (n > 0 && last_off[n] > last_off[0] && !last_tokens) throw std::invalid_argument("no window tokens");
    std::vector<SampleRow> rows;
    std::vector<int> row_of(n, -1);
    for (int i = 0; i < n; i++) {
      const int nl = last_off[i + 1] - last_off[i];
      if (sample_is_greedy(top_k[i], repetition_penalty[i], nl) || !sg_accepts(nl, top_k[i])) continue;
      row_of[i] = (int)rows.size();
      rows.push_back(SampleRow{slots[i], last_tokens + last_off[i], nl, repetition_penalty[i], top_k[i]});
    }
    std::vector<int> picks((size_t)2 * m->n_slots);
    Engine& e = *m->llm->engine;
    const SampleGpuOut* res = e.multi_sample(rows.data(), (int)rows.size(), picks.data());
    for (int i = 0; i < n; i++) {
      const int slot = slots[i];
      m->llm->rng.seed((unsigned)(seed[i] < 0 ? (int)time(nullptr) : seed[i]));
      bool used_device = false;
      out[i] = sample_lazy(
          m->llm->hp.n_vocab, last_tokens ? last_tokens + last_off[i] : nullptr, last_off[i + 1] - last_off[i], top_k[i], top_p[i], temperature[i],
          repetition_penalty[i], m->llm->rng, used_device, [&] { return picks[2 * slot + 1] == 1 ? picks[2 * slot] : -1; },
          [&](const int*, int, float, int, int* ids, float* lg) { return row_of[i] < 0 ? -1 : sg_take(res[row_of[i]], ids, lg); },
          [&] {
            multi_fetch(m, slot);
            return m->logits[slot];
          });
      if (used_device) m->device_samples++;
    }
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: multi-sequence sampling failed: %s\n", e.what());
    return -1;
  } catch (...) { return -1; }
}

long ctb_multi_device_samples(ctb_multi* m) { return m->device_samples; }

// the greedy pick of each slot: sample with top_k 1, top_p 1, temperature 1, no penalty
int ctb_multi_greedy(ctb_multi* m, int n, const int* slots, int* out) {
  if (n < 0) return -1;
  const std::vector<int> off(n + 1, 0), k(n, 1), seed(n, 0);
  const std::vector<float> one(n, 1.0f);
  return ctb_multi_sample_many(m, n, slots, off.data(), nullptr, k.data(), one.data(), one.data(), one.data(), seed.data(), out);
}

int ctb_multi_sample(ctb_multi* m, int slot, const int* last_tokens, int n_last, int top_k, float top_p, float temperature, float repetition_penalty,
                     int seed) {
  const int off[2] = {0, std::max(n_last, 0)};
  int tok = -1;
  return ctb_multi_sample_many(m, 1, &slot, off, last_tokens, &top_k, &top_p, &temperature, &repetition_penalty, &seed, &tok) == 0 ? tok : -1;
}

int ctb_multi_reset(ctb_multi* m, int slot) {
  try {
    if (!multi_slot_ok(m, slot)) return -1;
    m->llm->engine->multi_reset(slot);
    m->has[slot] = 0;
    m->fresh[slot] = 0;
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: multi-sequence reset failed: %s\n", e.what());
    return -1;
  }
}

size_t ctb_multi_state_size(ctb_multi* m, int n_tokens) {
  try { return state_size_for(*m->llm, n_tokens); } catch (...) { return 0; }
}

int ctb_multi_save(ctb_multi* m, int slot, const int* tokens, int n_tokens, void* buf, size_t cap) {
  try {
    if (!multi_slot_ok(m, slot)) return -1;
    save_state(*m->llm, slot, tokens, n_tokens, m->has[slot] != 0, buf, cap);
    return 0;
  } catch (const std::exception& e) { return state_error("cannot save the state", e); }
}

int ctb_multi_restore(ctb_multi* m, int slot, const void* buf, size_t size) {
  try {
    if (!multi_slot_ok(m, slot)) return -1;
    m->has[slot] = restore_state(*m->llm, slot, buf, size).has_results != 0;
    m->fresh[slot] = 0;
    return 0;
  } catch (const std::exception& e) { return state_error("cannot restore the state", e); }
}

int ctb_multi_fork(ctb_multi* m, int src, int n, const int* dsts) {
  try {
    if (!multi_slot_ok(m, src)) return -1;
    for (int i = 0; i < n; i++) {
      if (!multi_slot_ok(m, dsts[i])) return -1;
      if (dsts[i] == src) throw std::invalid_argument("slot " + std::to_string(src) + " cannot be forked into itself");
    }
    m->llm->engine->state_fork(src, dsts, n);
    for (int i = 0; i < n; i++) {
      const int d = dsts[i];
      m->has[d] = m->has[src];
      m->fresh[d] = m->fresh[src];
      if (m->fresh[src]) {
        m->logits[d] = m->logits[src];
        m->embd[d] = m->embd[src];
      }
    }
    return 0;
  } catch (const std::exception& e) { return state_error("cannot fork the slot", e); }
}

// ---- beam search (the reference's llama_beam_search, llama.cpp:4334-4579, driven as its examples/beam_search does)
//
// The reference keeps one KV cache: each step it evaluates the beams' common prefix as one chunk and shifts it off, then every
// beam's remaining tokens as one chunk, beam after beam.  Here each live beam owns a slot, and a step evaluates every live beam's
// newest token in one multi_eval.  What a chunk changes is the row length n_total of its V·P dots (DESIGN §2, item 4); the
// reference's f16 dot puts the elements below n_total & ~31 in its fp32 lanes and adds the rest one by one, and the entries
// past a token's own position are 0.  So a position p's K / V come out of one of two sums, told apart by vp_lanes(p, n_total).
// Each slot records the (token, sum) of every position it holds; a position whose sum differs from the reference's for this
// step is evaluated again, with every position after it.
static bool vp_lanes(int p, int n_total) { return (n_total & ~31) >= p + 1; }

struct SlotHeld { std::vector<int> tok; std::vector<char> lanes; };   // what a slot's K / V hold, per position

struct BeamRun {                  // one prompt's search
  int prompt = 0, P = 0;          // prompt index and length
  int c = 0;                      // tokens after the prompt shifted off as the beams' common prefix
  int iter = 0;
  std::vector<int> slots;         // its n_beams slots
  std::vector<BeamCand> beams, next;
  std::vector<std::vector<int>> toks;   // beams[i]'s tokens after the prompt
  std::vector<int> slot;                // beams[i]'s slot; -1 for an eob beam
  std::vector<int> fin_nt;              // the reference's n_total of positions P .. P + c - 1 (their common-prefix chunk)
};

// Appends a run of one slot's tokens at consecutive positions to a multi_eval list, cut into launches of MULTI_LAUNCH_TOKENS.
static void beam_append(std::vector<MultiTok>& toks, std::vector<int>& starts, int slot, const int* tokens, int pos0, const int* n_total, int n) {
  for (int j = 0; j < n; j++) {
    if ((int)toks.size() - starts.back() == MULTI_LAUNCH_TOKENS) starts.push_back((int)toks.size());
    toks.push_back({slot, tokens[j], pos0 + j, n_total[j], j == n - 1});
  }
}

int ctb_beam_step(int n_beams, int n_in, int n_next, const float* in_p, const unsigned char* in_eob, const float* rows, int n_vocab, int* out_parent,
                  int* out_token, float* out_p, unsigned char* out_eob) {
  try {
    if (n_beams < 1 || n_beams > n_vocab) throw std::invalid_argument("n_beams must lie in 1 .. n_vocab");
    if (n_in < 1 || n_in > n_beams || n_next < 0 || n_next > n_beams) throw std::invalid_argument("bad beam counts");
    std::vector<BeamCand> beams(n_in), next(n_next, BeamCand{0.0f, false, -1, -1});
    std::vector<const float*> r(n_in);
    for (int i = 0; i < n_in; i++) {
      beams[i] = {in_p[i], in_eob[i] != 0, -1, -1};
      r[i] = rows + (size_t)i * n_vocab;
    }
    const std::vector<BeamCand> out = beam_step(n_beams, beams, next, r.data(), n_vocab);
    for (size_t j = 0; j < out.size(); j++) {
      out_parent[j] = out[j].parent; out_token[j] = out[j].token; out_p[j] = out[j].p; out_eob[j] = out[j].eob;
    }
    return (int)out.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: beam step failed: %s\n", e.what());
    return -1;
  }
}

long ctb_multi_reparent(ctb_multi* m, int n, const int* src, const int* dst, const int* lo, const int* hi) {
  try {
    std::vector<KvCopy> copies(n);
    for (int i = 0; i < n; i++) {
      if (!multi_slot_ok(m, src[i]) || !multi_slot_ok(m, dst[i])) return -1;
      copies[i] = {src[i], dst[i], lo[i], hi[i]};
    }
    const size_t bytes = m->llm->engine->kv_reparent(copies);
    for (const KvCopy& c : copies) {
      m->has[c.dst] = m->has[c.src];
      m->fresh[c.dst] = 0;
    }
    return (long)bytes;
  } catch (const std::exception& e) { return state_error("cannot re-parent the slots", e); }
}

int ctb_multi_beam_search(ctb_multi* m, int n_prompts, const int* prompt_off, const int* prompt_tokens, int n_beams, int n_predict, int batch_size,
                          int* out_off, int* out_tokens, float* out_p) {
  using clk = std::chrono::steady_clock;
  const auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
  std::vector<char> used(m->n_slots, 0);
  try {
    const HParams& hp = m->llm->hp;
    const int n_vocab = hp.n_vocab, eos = m->llm->vocab.eos;
    if (n_prompts < 0) throw std::invalid_argument("a negative prompt count");
    if (n_beams < 1 || n_beams > m->n_slots) throw std::invalid_argument("n_beams = " + std::to_string(n_beams) + ": each beam needs a slot, and there are " + std::to_string(m->n_slots));
    if (n_beams > n_vocab) throw std::invalid_argument("n_beams is larger than the vocabulary");
    if (n_predict < 0) throw std::invalid_argument("a negative n_predict");
    for (int i = 0; i < n_prompts; i++) {
      const int P = prompt_off[i + 1] - prompt_off[i];
      if (P < 1) throw std::invalid_argument("prompt " + std::to_string(i) + " is empty");
      if (P + n_predict > hp.n_ctx)
        throw std::invalid_argument("prompt " + std::to_string(i) + ": " + std::to_string(P) + " tokens and " + std::to_string(n_predict) +
                                    " more exceed the context length " + std::to_string(hp.n_ctx));
      check_tokens(prompt_tokens + prompt_off[i], P, n_vocab);
    }
    double stats[8] = {0};   // ctb_multi_beam_stats
    out_off[0] = 0;
    std::vector<std::vector<int>> result(n_prompts);
    std::vector<float> result_p(n_prompts, 1.0f);
    Engine& e = *m->llm->engine;
    std::vector<SlotHeld> held(m->n_slots);
    std::vector<int> free_slots;
    for (int s = 0; s < m->n_slots; s++) free_slots.push_back(s);
    std::vector<BeamRun> runs;
    int waiting = n_predict > 0 ? 0 : n_prompts;   // (n_predict 0: the reference's loop never runs; the response is empty, p 1)
    std::vector<int> pos, nt;
    while (!runs.empty() || waiting < n_prompts) {
      std::vector<MultiTok> toks;
      std::vector<int> starts(1, 0);
      // the loop's test and the example's callback, then each live beam's tokens whose K / V differ from the reference's
      for (size_t r = 0; r < runs.size();) {
        BeamRun& R = runs[r];
        const bool any_live = std::any_of(R.beams.begin(), R.beams.end(), [](const BeamCand& b) { return !b.eob; });
        if (!(R.iter < n_predict && any_live && !R.beams[beam_top(R.beams)].eob)) {
          const size_t top = beam_top(R.beams);   // collapse; the last callback collects the rest of the top beam's tokens
          result[R.prompt] = R.toks[top];
          result_p[R.prompt] = R.beams[top].p;
          free_slots.insert(free_slots.end(), R.slots.begin(), R.slots.end());
          runs.erase(runs.begin() + r);
          continue;
        }
        const size_t nb = R.beams.size();
        for (size_t i = 0; i < nb; i++)
          if (!R.beams[i].eob && !R.toks[i].empty() && R.toks[i].back() == eos) {
            R.beams[i].eob = true;
            R.slot[i] = -1;   // an eob beam is never evaluated again: its slot is free
          }
        size_t cpl = R.toks[0].size() - R.c;
        for (size_t i = 1; i < nb; i++) {
          cpl = std::min(cpl, R.toks[i].size() - R.c);
          for (size_t j = 0; j < cpl; j++)
            if (R.toks[i][R.c + j] != R.toks[0][R.c + j]) { cpl = j; break; }
        }
        for (size_t j = 0; j < cpl; j++) R.fin_nt.push_back(R.P + R.c + (int)cpl);
        R.c += (int)cpl;
        for (size_t i = 0; i < nb; i++) {
          if (R.beams[i].eob) continue;
          const std::vector<int>& t = R.toks[i];
          const int L = (int)t.size(), s = R.slot[i];
          SlotHeld& h = held[s];
          nt.resize(L);
          for (int j = 0; j < L; j++) nt[j] = j < R.c ? R.fin_nt[j] : R.P + L;
          int q = L - 1;   // the newest token always runs: its row is this step's
          for (int j = 0; j < L - 1; j++)
            if (R.P + j >= (int)h.tok.size() || h.tok[R.P + j] != t[j] || h.lanes[R.P + j] != vp_lanes(R.P + j, nt[j])) { q = j; break; }
          h.tok.resize(R.P + q); h.lanes.resize(R.P + q);
          for (int j = q; j < L; j++) { h.tok.push_back(t[j]); h.lanes.push_back(vp_lanes(R.P + j, nt[j])); }
          beam_append(toks, starts, s, t.data() + q, R.P + q, nt.data() + q, L - q);
        }
        r++;
      }
      // admission: a prompt takes n_beams free slots and is evaluated, chunked as LLM::BatchEval chunks it, in the first
      bool admitted = false;
      while (waiting < n_prompts && (int)free_slots.size() >= n_beams) {
        std::sort(free_slots.begin(), free_slots.end());
        BeamRun R;
        R.prompt = waiting++;
        R.P = prompt_off[R.prompt + 1] - prompt_off[R.prompt];
        R.slots.assign(free_slots.begin(), free_slots.begin() + n_beams);
        free_slots.erase(free_slots.begin(), free_slots.begin() + n_beams);
        for (int s : R.slots) {
          e.multi_reset(s);
          used[s] = 1;
          m->has[s] = 0; m->fresh[s] = 0;
          held[s] = SlotHeld();
        }
        const int* pt = prompt_tokens + prompt_off[R.prompt];
        pos.resize(R.P); nt.resize(R.P);
        eval_positions(R.P, 0, batch_size, hp.n_ctx, pos.data(), nt.data());
        SlotHeld& h = held[R.slots[0]];
        for (int j = 0; j < R.P; j++) {
          h.tok.push_back(pt[j]);
          h.lanes.push_back(vp_lanes(pos[j], nt[j]));
        }
        beam_append(toks, starts, R.slots[0], pt, 0, nt.data(), R.P);
        R.beams.push_back(BeamCand{1.0f, false, -1, -1});
        R.toks.emplace_back();
        R.slot.push_back(R.slots[0]);
        runs.push_back(std::move(R));
        admitted = true;
      }
      if (runs.empty()) continue;
      // one batched eval of every live beam's tokens (and of the prompts just admitted)
      auto t0 = clk::now();
      if ((int)toks.size() > starts.back()) starts.push_back((int)toks.size());
      if (!toks.empty()) {
        e.multi_eval(toks, starts);
        for (const MultiTok& t : toks) { m->has[t.slot] = 1; m->fresh[t.slot] = 0; }
      }
      auto t1 = clk::now();
      // their logits rows in one copy, then the reference's selection
      int lo_s = m->n_slots, hi_s = -1;
      for (const BeamRun& R : runs)
        for (size_t i = 0; i < R.beams.size(); i++)
          if (!R.beams[i].eob) { lo_s = std::min(lo_s, R.slot[i]); hi_s = std::max(hi_s, R.slot[i]); }
      const float* rows = hi_s >= lo_s ? e.multi_rows(lo_s, hi_s - lo_s + 1) : nullptr;
      std::vector<KvCopy> copies;
      for (BeamRun& R : runs) {
        std::vector<const float*> rp(R.beams.size(), nullptr);
        for (size_t i = 0; i < R.beams.size(); i++)
          if (!R.beams[i].eob) rp[i] = rows + (size_t)(R.slot[i] - lo_s) * n_vocab;
        std::vector<BeamCand> nb = beam_step(n_beams, R.beams, R.next, rp.data(), n_vocab);
        // Slots of the new beams.  A live parent's first child keeps the parent's slot; every other child takes a slot that no
        // kept parent holds (a parent without children, an eob beam's, one not used yet).  So the copies' sources (kept slots)
        // and destinations (the others) are disjoint, and one launch can run them all: no copy reads a slot another writes.
        std::vector<int> slot(nb.size(), -1);
        std::vector<std::vector<int>> nt_toks(nb.size());
        std::vector<char> kept(m->n_slots, 0);
        for (size_t j = 0; j < nb.size(); j++) {
          const int pa = nb[j].parent;
          nt_toks[j] = R.toks[pa];
          if (nb[j].token < 0) continue;
          nt_toks[j].push_back(nb[j].token);
          if (!kept[R.slot[pa]]) { kept[R.slot[pa]] = 1; slot[j] = R.slot[pa]; }
        }
        std::vector<int> spare;
        for (int s : R.slots)
          if (!kept[s]) spare.push_back(s);
        for (size_t j = 0; j < nb.size(); j++) {
          if (nb[j].token < 0 || slot[j] >= 0) continue;
          if (spare.empty()) throw std::logic_error("beam search: more live beams than slots");
          const int src = R.slot[nb[j].parent], dst = spare.back();
          spare.pop_back();
          const SlotHeld &hs = held[src], &hd = held[dst];
          int lo = 0;
          while (lo < (int)std::min(hs.tok.size(), hd.tok.size()) && hs.tok[lo] == hd.tok[lo] && hs.lanes[lo] == hd.lanes[lo]) lo++;
          copies.push_back({src, dst, lo, (int)hs.tok.size()});
          held[dst] = hs;
          slot[j] = dst;
        }
        R.next = std::move(R.beams);
        R.beams = std::move(nb);
        R.toks = std::move(nt_toks);
        R.slot = std::move(slot);
        R.iter++;
      }
      auto t2 = clk::now();
      // one re-parenting launch for every prompt's copies
      stats[4] += (double)e.kv_reparent(copies);
      for (const KvCopy& c : copies) { m->has[c.dst] = m->has[c.src]; m->fresh[c.dst] = 0; }
      auto t3 = clk::now();
      stats[0] += 1; stats[1] += ms(t0, t1); stats[2] += ms(t1, t2); stats[3] += ms(t2, t3); stats[5] += (double)toks.size();
      if (admitted) { stats[6] += 1; stats[7] += ms(t0, t1); }
    }
    for (int s = 0; s < m->n_slots; s++)
      if (used[s]) ctb_multi_reset(m, s);
    for (int i = 0; i < n_prompts; i++) {
      out_off[i + 1] = out_off[i] + (int)result[i].size();
      std::copy(result[i].begin(), result[i].end(), out_tokens + out_off[i]);
      out_p[i] = result_p[i];
    }
    std::copy(stats, stats + 8, m->beam_stats);
    return 0;
  } catch (const std::exception& ex) {
    fprintf(stderr, "ctransformers-b200: beam search failed: %s\n", ex.what());
    try {
      for (int s = 0; s < m->n_slots; s++)
        if (used[s]) ctb_multi_reset(m, s);
    } catch (...) {}
    return -1;
  }
}

int ctb_multi_beam_stats(ctb_multi* m, double* out8) {
  std::copy(m->beam_stats, m->beam_stats + 8, out8);
  return 8;
}

long ctb_multi_launches(ctb_multi* m) { return m->llm->engine->multi_launches(); }
double ctb_multi_last_eval_ms(ctb_multi* m) { return m->llm->engine->stats.last_eval_ms; }

int ctb_multi_pack(int n, const int* slots, const int* off, const int* n_past, int batch_size, int n_ctx, int* out, int cap) {
  try {
    std::vector<MultiTok> toks;
    const std::vector<int> starts = multi_pack(n, slots, off, nullptr, n_past, batch_size, n_ctx, toks);
    if ((int)toks.size() > cap) return -(int)toks.size();
    for (size_t l = 0; l + 1 < starts.size(); l++)
      for (int i = starts[l]; i < starts[l + 1]; i++) {
        const MultiTok& t = toks[i];
        int* o = out + (size_t)i * 5;
        o[0] = t.slot; o[1] = t.pos; o[2] = t.n_total; o[3] = (int)l; o[4] = t.last ? 1 : 0;
      }
    return (int)toks.size();
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: %s\n", e.what());
    return 0;
  }
}

int ctb_sample(const float* logits, int n_vocab, const int* last_tokens, int n_last, int top_k, float top_p, float temperature,
               float repetition_penalty, int seed) {
  try {
    if (seed < 0) seed = (int)time(nullptr);
    std::mt19937 rng((unsigned)seed);
    return sample_token(logits, n_vocab, last_tokens, n_last, top_k, top_p, temperature, repetition_penalty, rng);
  } catch (...) { return -1; }
}

}  // extern "C"

// ----------------------------------------------------------------------------- grammar-constrained sampling
struct ctb_grammar { std::shared_ptr<const Grammar> g; };
struct ctb_grammar_state { std::shared_ptr<const Grammar> g; GrammarState s; };

ctb_grammar* ctb_grammar_parse(const char* text, char* err, int cap, long* err_pos) {
  auto report = [&](const std::string& m, long pos) {
    if (err && cap > 0) { const size_t n = std::min(m.size(), (size_t)cap - 1); memcpy(err, m.data(), n); err[n] = 0; }
    if (err_pos) *err_pos = pos;
  };
  try {
    if (!text) throw GrammarError("no grammar text", 0);
    std::unique_ptr<ctb_grammar> g(new ctb_grammar);
    g->g = std::make_shared<const Grammar>(grammar_parse(text));
    report("", -1);
    return g.release();
  } catch (const GrammarError& e) {
    report(e.what(), e.pos);
  } catch (const std::exception& e) {
    report(e.what(), 0);
  }
  return nullptr;
}
void ctb_grammar_free(ctb_grammar* g) { delete g; }
int ctb_grammar_info(const ctb_grammar* g, int* out3) {
  out3[0] = g->g->n_rules(); out3[1] = (int)g->g->elems.size(); out3[2] = (int)g->g->symbols.size();
  return 3;
}
int ctb_grammar_rules(const ctb_grammar* g, int* off, unsigned* elems) {
  std::copy(g->g->off.begin(), g->g->off.end(), off);
  for (size_t i = 0; i < g->g->elems.size(); i++) { elems[2 * i] = g->g->elems[i].type; elems[2 * i + 1] = g->g->elems[i].value; }
  return g->g->n_rules();
}
int ctb_grammar_symbol(const ctb_grammar* g, int i, char* name, int cap, unsigned* id) {
  if (i < 0 || i >= (int)g->g->symbols.size()) return 0;
  const auto& s = g->g->symbols[i];
  *id = s.second;
  if ((int)s.first.size() > cap) return -(int)s.first.size();
  memcpy(name, s.first.data(), s.first.size());
  return (int)s.first.size();
}
ctb_grammar_state* ctb_grammar_start(const ctb_grammar* g) {
  try { return new ctb_grammar_state{g->g, grammar_start(*g->g)}; } catch (...) { return nullptr; }
}
ctb_grammar_state* ctb_grammar_state_copy(const ctb_grammar_state* s) {
  try { return new ctb_grammar_state(*s); } catch (...) { return nullptr; }
}
void ctb_grammar_state_free(ctb_grammar_state* s) { delete s; }
int ctb_grammar_state_eos_ok(const ctb_grammar_state* s) { return s->s.eos_ok() ? 1 : 0; }
int ctb_grammar_state_stacks(const ctb_grammar_state* s, int* out, int cap, int* partial2) {
  std::vector<int> v;   // per stack: its length, then its elements bottom first
  for (const auto& st : s->s.stacks) { v.push_back((int)st.size()); v.insert(v.end(), st.begin(), st.end()); }
  partial2[0] = (int)s->s.partial.value;
  partial2[1] = s->s.partial.n_remain;
  if ((int)v.size() > cap) return -(int)v.size();
  std::copy(v.begin(), v.end(), out);
  return (int)v.size();
}

static int grammar_accept_or_refuse(ctb_grammar_state* s, bool is_eos, const std::string& piece) {
  try {
    grammar_accept(*s->g, s->s, is_eos, piece);
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: grammar accept failed: %s\n", e.what());
    return -1;
  }
}
int ctb_grammar_accept_piece(ctb_grammar_state* s, const char* piece, int len, int is_eos) {
  return grammar_accept_or_refuse(s, is_eos != 0, std::string(piece ? piece : "", piece ? std::max(len, 0) : 0));
}
static int llm_grammar_accept(LLM* llm, ctb_grammar_state* s, int token) {
  if (token < 0 || token >= llm->hp.n_vocab) {
    fprintf(stderr, "ctransformers-b200: grammar accept failed: token %d is out of range\n", token);
    return -1;
  }
  return grammar_accept_or_refuse(s, token == llm->vocab.eos, token == llm->vocab.eos ? std::string() : llm->vocab.piece(token));
}
int ctb_llm_grammar_accept(LLM* llm, ctb_grammar_state* s, int token) { return llm_grammar_accept(llm, s, token); }
int ctb_multi_grammar_accept(ctb_multi* m, ctb_grammar_state* s, int token) { return llm_grammar_accept(m->llm.get(), s, token); }

int ctb_grammar_mask_pieces(const ctb_grammar_state* s, int n_vocab, const int* off, const char* bytes, int eos, unsigned char* allowed) {
  try {
    grammar_mask(*s->g, s->s, n_vocab, eos, [&](int t) { return std::string(bytes + off[t], bytes + off[t + 1]); }, allowed);
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: grammar mask failed: %s\n", e.what());
    return -1;
  }
}

// the host mask over the model's vocabulary
static void host_mask(LLM* llm, const ctb_grammar_state* s, uint8_t* allowed) {
  grammar_mask(*s->g, s->s, llm->hp.n_vocab, llm->vocab.eos, [&](int t) { return llm->vocab.piece(t); }, allowed);
}

// The rows below hold logits after the repetition penalty and the grammar mask (llama.cc:53-84 with llama_sample_grammar
// between the penalty and top-k, as examples/main/main.cpp:650-695 places it): the host version of what k_grammar_mask writes.
static std::vector<float> host_masked(LLM* llm, std::vector<float> v, const int* last, int n_last, float penalty, const ctb_grammar_state* s) {
  if (n_last > 0 && penalty != 1.0f)
    for (size_t i = 0; i < v.size(); i++) {
      if (std::find(last, last + n_last, (int)i) == last + n_last) continue;
      if (v[i] <= 0) v[i] *= penalty; else v[i] /= penalty;
    }
  std::vector<uint8_t> ok(v.size());
  host_mask(llm, s, ok.data());
  size_t n_ok = 0;
  for (size_t i = 0; i < v.size(); i++) {
    if (!ok[i]) v[i] = -INFINITY;
    n_ok += ok[i];
  }
  if (!n_ok) throw std::invalid_argument("the grammar allows no token here");
  return v;
}

static void grammar_pieces_once(LLM* llm) {
  Engine& e = *llm->engine;
  if (e.has_grammar_pieces()) return;
  std::vector<int> off(1, 0);
  std::vector<uint8_t> bytes;
  for (int t = 0; t < llm->hp.n_vocab; t++) {
    const std::string p = llm->vocab.piece(t);
    const size_t n = std::find(p.begin(), p.end(), '\0') - p.begin();   // the reference decodes the piece as a C string
    bytes.insert(bytes.end(), p.begin(), p.begin() + n);
    off.push_back((int)bytes.size());
  }
  e.grammar_pieces(off, bytes);
}

// The device's top-k cut of a constrained row: its candidates' count (ids / logits filled), or -1 when the row has fewer allowed
// tokens than the cut (equal -inf keys make the cut ambiguous) or the device took no cut.
static int grammar_cut(const SampleGpuOut& res, int allowed, int top_k, int V, int* ids, float* lg) {
  return sg_accepts(0, top_k) && allowed >= std::min(std::max(top_k, 1), V) ? sg_take(res, ids, lg) : -1;
}
// whether the draw of a row the device finished takes the host sampler on its masked row (sample_lazy's test)
static bool grammar_needs_host_cut(const SampleGpuOut& res, int allowed, int top_k, int V) {
  int ids[SG_MAX_OUT];
  float lg[SG_MAX_OUT];
  std::vector<Candidate> c;
  const int count = grammar_cut(res, allowed, top_k, V, ids, lg);
  return !(count > 0 && device_candidates_usable(ids, lg, count, top_k, V, c));
}

// One constrained draw from the device's results for its row: the device's top-k cut when it is usable (as many allowed tokens as
// the cut and an unambiguous cut), else the host sampler on the masked row (scratch: that row when the caller fetched it already);
// a row the device could not finish is masked on the host from the slot's logits.
static int grammar_draw(LLM* llm, long* paths, int r, int slot, const int* stats, const SampleGpuOut& res, const int* last, int n_last, int top_k,
                        float top_p, float temperature, float penalty, const ctb_grammar_state* s, const std::vector<float>* scratch = nullptr) {
  Engine& e = *llm->engine;
  const int V = llm->hp.n_vocab;
  if (stats[2 * r + 1]) {
    paths[1]++;
    const std::vector<float> v = host_masked(llm, e.slot_logits(slot), last, n_last, penalty, s);
    return sample_token(v.data(), V, nullptr, 0, top_k, top_p, temperature, 1.0f, llm->rng);
  }
  const int allowed = stats[2 * r];
  if (allowed == 0) throw std::invalid_argument("the grammar allows no token here");
  bool used_device = false;
  const int t = sample_lazy(
      V, nullptr, 0, top_k, top_p, temperature, 1.0f, llm->rng, used_device, [] { return -1; },
      [&](const int*, int, float, int, int* ids, float* lg) { return grammar_cut(res, allowed, top_k, V, ids, lg); },
      [&] { return scratch ? *scratch : std::move(e.grammar_scratch({r})[0]); });
  paths[used_device ? 0 : 2]++;
  return t;
}

int ctb_llm_sample_grammar(LLM* llm, const int* last_tokens, int n_last, int top_k, float top_p, float temperature, float repetition_penalty,
                           int seed, const ctb_grammar_state* s) {
  try {
    not_sharded(llm, "does not sample with a grammar");
    if (!s) throw std::invalid_argument("no grammar state");
    if (!llm->has_logits) throw std::invalid_argument("nothing has been evaluated");
    if (n_last > 0 && !last_tokens) throw std::invalid_argument("no window tokens");
    if (seed < 0) seed = (int)time(nullptr);
    llm->rng.seed((unsigned)seed);
    Engine& e = *llm->engine;
    if (!e.lazy_logits()) {
      // a host view of the logits is held (and may have been changed by the caller): mask on the host over that view
      const float* view = e.logits();
      const std::vector<float> v = host_masked(llm, std::vector<float>(view, view + llm->hp.n_vocab), last_tokens, n_last, repetition_penalty, s);
      llm->grammar_paths[2]++;
      return sample_token(v.data(), llm->hp.n_vocab, nullptr, 0, top_k, top_p, temperature, 1.0f, llm->rng);
    }
    grammar_pieces_once(llm);
    const GrammarRow row{0, s->g.get(), &s->s, last_tokens, n_last, repetition_penalty, sg_accepts(0, top_k) ? top_k : 0};
    int stats[2];
    const SampleGpuOut* res = e.grammar_rows(&row, 1, llm->vocab.eos, stats);
    return grammar_draw(llm, llm->grammar_paths, 0, 0, stats, res[0], last_tokens, n_last, top_k, top_p, temperature, repetition_penalty, s);
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: grammar sampling failed: %s\n", e.what());
    return -1;
  } catch (...) { return -1; }
}

// the device mask of a state on one slot's engine; a row the device could not finish is masked on the host
static int engine_mask(LLM* llm, long* paths, int slot, const ctb_grammar_state* s, unsigned char* allowed) {
  try {
    not_sharded(llm, "does not sample with a grammar");
    if (!s || !allowed) throw std::invalid_argument("a missing argument");
    grammar_pieces_once(llm);
    const int V = llm->hp.n_vocab;
    const GrammarRow row{slot, s->g.get(), &s->s, nullptr, 0, 1.0f, 0};
    int stats[2];
    std::vector<unsigned> bits((size_t)(V + 31) / 32);
    llm->engine->grammar_rows(&row, 1, llm->vocab.eos, stats, bits.data());
    if (stats[1]) {
      paths[1]++;
      host_mask(llm, s, allowed);
      return 0;
    }
    for (int t = 0; t < V; t++) allowed[t] = (bits[t / 32] >> (t % 32)) & 1u;
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: grammar mask failed: %s\n", e.what());
    return -1;
  } catch (...) { return -1; }
}
int ctb_llm_grammar_mask(LLM* llm, const ctb_grammar_state* s, unsigned char* allowed) {
  return engine_mask(llm, llm->grammar_paths, 0, s, allowed);
}
int ctb_multi_grammar_mask(ctb_multi* m, int slot, const ctb_grammar_state* s, unsigned char* allowed) {
  if (!multi_slot_ok(m, slot)) return -1;
  return engine_mask(m->llm.get(), m->llm->grammar_paths, slot, s, allowed);
}

int ctb_multi_sample_grammar_many(ctb_multi* m, int n, const int* slots, const int* last_off, const int* last_tokens, const int* top_k,
                                  const float* top_p, const float* temperature, const float* repetition_penalty, const int* seed,
                                  const ctb_grammar_state* const* states, int* out) {
  try {
    if (n < 0) throw std::invalid_argument("a negative slot count");
    if (n > 0 && (!slots || !last_off || !top_k || !top_p || !temperature || !repetition_penalty || !seed || !out || !states))
      throw std::invalid_argument("a missing argument array");
    if (!multi_slots_ok(m, n, slots)) return -1;
    for (int i = 0; i < n; i++) {
      if (!m->has[slots[i]]) throw std::invalid_argument("slot " + std::to_string(slots[i]) + " has no logits to sample from");
      if (last_off[i] < 0 || last_off[i + 1] < last_off[i]) throw std::invalid_argument("the window offsets of slot " + std::to_string(slots[i]) + " are not ascending");
    }
    if (n > 0 && last_off[n] > last_off[0] && !last_tokens) throw std::invalid_argument("no window tokens");
    // the unconstrained draws: exactly ctb_multi_sample_many on them
    std::vector<int> free_i, u_slots, u_off(1, 0), u_last, u_k, u_seed, u_out;
    std::vector<float> u_p, u_t, u_pen;
    std::vector<GrammarRow> rows;
    std::vector<int> row_i;
    for (int i = 0; i < n; i++) {
      const int* w = last_tokens ? last_tokens + last_off[i] : nullptr;
      const int nl = last_off[i + 1] - last_off[i];
      if (states[i]) {
        rows.push_back(GrammarRow{slots[i], states[i]->g.get(), &states[i]->s, w, nl, repetition_penalty[i], sg_accepts(0, top_k[i]) ? top_k[i] : 0});
        row_i.push_back(i);
        continue;
      }
      free_i.push_back(i);
      u_slots.push_back(slots[i]);
      if (nl > 0) u_last.insert(u_last.end(), w, w + nl);
      u_off.push_back((int)u_last.size());
      u_k.push_back(top_k[i]); u_p.push_back(top_p[i]); u_t.push_back(temperature[i]); u_pen.push_back(repetition_penalty[i]);
      u_seed.push_back(seed[i]);
    }
    if (!free_i.empty()) {
      u_out.resize(free_i.size());
      if (ctb_multi_sample_many(m, (int)free_i.size(), u_slots.data(), u_off.data(), u_last.data(), u_k.data(), u_p.data(), u_t.data(), u_pen.data(),
                                u_seed.data(), u_out.data()) != 0)
        return -1;
      for (size_t j = 0; j < free_i.size(); j++) out[free_i[j]] = u_out[j];
    }
    if (rows.empty()) return 0;
    LLM& L = *m->llm;
    grammar_pieces_once(&L);
    std::vector<int> stats(2 * rows.size());
    const SampleGpuOut* res = L.engine->grammar_rows(rows.data(), (int)rows.size(), L.vocab.eos, stats.data());
    std::vector<SampleGpuOut> results(res, res + rows.size());
    // the masked rows the host cuts come back together: one copy each, one synchronise
    std::vector<int> host_rows, at(rows.size(), -1);
    for (size_t r = 0; r < rows.size(); r++)
      if (!stats[2 * r + 1] && stats[2 * r] > 0 && grammar_needs_host_cut(results[r], stats[2 * r], top_k[row_i[r]], L.hp.n_vocab)) {
        at[r] = (int)host_rows.size();
        host_rows.push_back((int)r);
      }
    const std::vector<std::vector<float>> scratch = host_rows.empty() ? std::vector<std::vector<float>>() : L.engine->grammar_scratch(host_rows);
    for (size_t r = 0; r < rows.size(); r++) {
      const int i = row_i[r];
      L.rng.seed((unsigned)(seed[i] < 0 ? (int)time(nullptr) : seed[i]));
      out[i] = grammar_draw(&L, L.grammar_paths, (int)r, slots[i], stats.data(), results[r], rows[r].last, rows[r].n_last, top_k[i], top_p[i],
                            temperature[i], repetition_penalty[i], states[i], at[r] >= 0 ? &scratch[at[r]] : nullptr);
    }
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: multi-sequence grammar sampling failed: %s\n", e.what());
    return -1;
  } catch (...) { return -1; }
}

int ctb_llm_grammar_paths(LLM* llm, long* out3) { std::copy(llm->grammar_paths, llm->grammar_paths + 3, out3); return 3; }
int ctb_multi_grammar_paths(ctb_multi* m, long* out3) { return ctb_llm_grammar_paths(m->llm.get(), out3); }
