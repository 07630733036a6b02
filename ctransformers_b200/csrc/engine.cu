// See engine.cuh.  Model upload (GGUF blocks → device planes), tables, KV cache, op schedule, CUDA graphs.
#include "engine.cuh"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include "attention.cuh"
#include "grammar.hpp"
#include "grammar_gpu.cuh"
#include "matvec.cuh"
#include "prefill.cuh"
#include "repack.cuh"
#include "sample_gpu.cuh"
#include "score_gpu.cuh"
#include "stream.cuh"
#include "tables.hpp"
#include "tp_nccl.hpp"

namespace ctb {

#define CTB_CUDA(expr)                                                                                         \
  do {                                                                                                         \
    cudaError_t e__ = (expr);                                                                                  \
    if (e__ != cudaSuccess)                                                                                    \
      throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(e__) + " at " + __FILE__ + ":" + \
                               std::to_string(__LINE__) + " (" #expr ")" + watchdog_note());                   \
  } while (0)

// what a trapped persistent kernel left in the host-mapped watchdog words (stream.cuh st_fail)
static int* g_watchdog_words = nullptr;
static std::string watchdog_note() {
  const int* d = g_watchdog_words;
  if (!d) return " [no watchdog words]";
  if (d[0] == 0) return " [watchdog words clear]";
  const char* w = (d[0] > 0 && d[0] < W_CODES) ? WAIT_TEXT[d[0]] : "?";
  return " [step-kernel watchdog: wait " + std::to_string(d[0]) + " (" + w + ") timed out in CTA " + std::to_string(d[1]) + ", aux " + std::to_string(d[2]) + ", thread " +
         std::to_string(d[3]) + "]";
}

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// the engine works on its own device but leaves the caller's current device as it found it
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) {
      cudaError_t e = cudaSetDevice(dev);
      if (e != cudaSuccess) throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(e) + " (cudaSetDevice)");
    }
  }
  ~DeviceGuard() { int cur = -1; cudaGetDevice(&cur); if (prev >= 0 && cur != prev) cudaSetDevice(prev); }
};

// one op of the per-token schedule: a phase of the step kernel, or (mat-vecs over non-K-quant weights) a kernel of its own
struct StepOp {
  Phase ph;
  int mvk = 0;          // PH_MATVEC: which projection (MVK_*)
  bool stream = false;  // PH_MATVEC: runs inside the step kernel
};

// advance the on-device decode state after k_argmax's greedy pick (state[4])
__global__ void k_advance(int* state, int* out_tokens) { advance_state(state, out_tokens, state[4]); }

// ---- batched prefill (prefill.cuh): the per-token schedule rewritten over PB_T-row buffers, as one program of k_pstep: the
// body, then, when the output head is a K-quant, its QUANT + GEMM phases over every token of the launch (logits rows in
// Engine::d_rows_, embeddings rows in embd_rows).  A launch runs the body alone or the whole program.
struct PrefillState {
  std::vector<DevMem> bufs;         // the batched buffers and the QUANT phases' scratch (dalloc)
  std::vector<PPhase> phases;
  DevMem d_phases;                  // their device copy (zeroed one phase past the end)
  int n_body = 0;                   // phases of the body: all of them when the head has no phases here
  bool q3_body = false, q3_all = false;   // the body / the whole program holds Q3_K matrices: the k_pstep<true> build
  int* d_state = nullptr;           // PB_STATE_MS ints: [PB_T][4] + n_tok, the slot strides, each token's slot (PB_S)
  StateRing ring;                   // d_state of each launch, PF_RING launches deep
  float* x_final = nullptr;         // batched buffer that holds the last layer's output rows
  float* embd_rows = nullptr;       // [PB_T][n_embd]: the head's QUANT phase writes every token's embeddings (the MS builds)
  int n_slots = 0;
  size_t smem = 0;
  bool ok = false, tried = false;
  long m_launches = 0;              // multi-sequence launches
  void* dalloc(size_t bytes) {      // zeroed device memory, freed with the state
    bufs.emplace_back(bytes);
    CTB_CUDA(cudaMemset(bufs.back().get(), 0, bytes));
    return bufs.back().get();
  }
  bool head() const { return n_body < (int)phases.size(); }
  cudaError_t launch(bool whole, int grid, cudaStream_t st, unsigned* d_sync, bool multi) const {
    return launch_pstep(grid, n_slots, smem, st, d_phases.as<PPhase>(), whole ? (int)phases.size() : n_body, d_sync, whole ? q3_all : q3_body, multi);
  }
};
constexpr int PF_RING = 64;
static_assert(MULTI_LAUNCH_TOKENS == PB_T, "multi_pack cuts launches of PB_T tokens");

constexpr size_t UP_CHUNK = (size_t)32 << 20;   // upload pipeline: chunk bytes and buffers in flight
constexpr int UP_BUFS = 3;

static bool supported_matrix_type(uint32_t t) {
  return t == T_F32 || t == T_F16 || t == T_Q4_0 || t == T_Q4_1 || t == T_Q5_0 || t == T_Q5_1 || t == T_Q8_0 || t == T_Q3_K || t == T_Q4_K || t == T_Q5_K ||
         t == T_Q6_K;
}

size_t engine_arena_bytes(const GGUFFile& g, const HParams& hp) {
  size_t total = 0;
  for (const auto& t : g.tensors) {
    total += align_up(t.nbytes, 256) + 4 * 256;   // up to 4 planes, each 256-aligned
    if (t.ne[1] > 0) total += align_up(t.nbytes / (size_t)t.ne[1] * ST_ROWS, 256);   // K-quants: rows padded to whole 16-row tiles
  }
  total += UP_CHUNK * UP_BUFS + 256;                                            // device staging of the upload pipeline
  const size_t kv = (size_t)hp.n_layer * (hp.n_ctx + 256) * hp.n_head_kv * k_stride(hp.head_dim()) * 2;   // K rows padded to 8 halves
  total += 2 * align_up(kv * hp.n_seq, 256);
  total += 3 * align_up(65536 * 2, 256);
  total += align_up((size_t)hp.n_ctx * (hp.head_dim() / 2) * 8, 256);
  const size_t qkv = (size_t)hp.n_embd + 2 * (size_t)hp.n_embd_gqa();
  total += 4 * (2 * (size_t)hp.n_embd + qkv + 3 * (size_t)hp.n_embd + 2 * (size_t)hp.n_ff + (size_t)hp.n_vocab) + 64 * 256 + 8192;
  total += (size_t)hp.n_seq * (4 * ((size_t)hp.n_vocab + hp.n_embd) + 8) + 256;   // every slot's kept results
  total += ((size_t)hp.n_layer * 10 + 8) * (sizeof(Phase) * 2 + 2 * 1024) + 8192;   // the step programs and their per-CTA tile ranges
  total += 1 << 20;
  return total;
}

void* Engine::alloc(size_t bytes, size_t align) {
  const size_t off = align_up(arena_used_, align);
  if (off + bytes > arena_size_) throw std::runtime_error("device arena exhausted");
  arena_used_ = off + bytes;
  return arena_.as<uint8_t>() + off;
}

// ---- load pipeline (reference: llama_model_loader::load_all_data, llama.cpp:1417-1487 + ggml_cuda_transform_tensor,
// ggml-cuda.cu:6359-6432 — a blocking cudaMemcpy per tensor).  Here a tensor travels in row chunks of <= UP_CHUNK bytes through
// UP_BUFS pinned host buffers and as many device staging buffers: the host thread copies chunk i+1 out of the mmap'ed file
// into pinned memory while chunk i is on the wire (cudaMemcpyAsync from pinned memory is truly asynchronous) and chunk i-1 is
// being repacked on the GPU; buffers are recycled behind events, nothing synchronises per tensor.
struct Uploader {
  HostMem host[UP_BUFS];
  uint8_t* dev[UP_BUFS] = {nullptr, nullptr, nullptr};
  Event done[UP_BUFS];
  Stream st[UP_BUFS];   // (declared after the buffers: a stream's work is done before they are freed)
  int next = 0;
  size_t bytes = 0;
  void init(uint8_t* dev_base) {
    for (int i = 0; i < UP_BUFS; i++) {
      host[i] = HostMem(UP_CHUNK);
      dev[i] = dev_base + (size_t)i * UP_CHUNK;
      done[i] = Event(cudaEventDisableTiming);
      st[i] = Stream(cudaStreamNonBlocking);
    }
  }
  // copies [src, src+n) to the device staging buffer of the next slot; returns the slot (its stream carries the copy)
  int push(const uint8_t* src, size_t n) {
    const int i = next;
    next = (next + 1) % UP_BUFS;
    CTB_CUDA(cudaEventSynchronize(done[i]));        // the slot's previous chunk has been repacked
    memcpy(host[i].get(), src, n);
    CTB_CUDA(cudaMemcpyAsync(dev[i], host[i].get(), n, cudaMemcpyHostToDevice, st[i]));
    bytes += n;
    return i;
  }
  void finish(int i) { CTB_CUDA(cudaEventRecord(done[i], st[i])); }
  void drain() { for (int i = 0; i < UP_BUFS; i++) CTB_CUDA(cudaStreamSynchronize(st[i])); }
};

// rows [row0, row1) and elements [k0, k1) of every row (whole quantization blocks) are kept: a tensor-parallel shard
// (column-parallel = a row range, row-parallel = a K range); the defaults keep the whole tensor.
DevMat Engine::upload_matrix(const GGUFTensor& t, Uploader& up, int want_K, int want_M, int row0, int row1, int k0, int k1) {
  if (!supported_matrix_type(t.type)) throw std::runtime_error("tensor '" + t.name + "': quantization type " + std::to_string(t.type) + " is not supported by the CUDA path");
  DevMat m;
  m.type = (int)t.type;
  const int full_K = (int)t.ne[0], full_M = (int)(t.ne[1] * t.ne[2] * t.ne[3]);
  // the reference rejects a tensor whose shape does not follow from the hyper-parameters (llama.cpp:1345-1361 "wrong shape")
  if (full_K != want_K || full_M != want_M)
    throw std::runtime_error("tensor '" + t.name + "' has wrong shape; expected " + std::to_string(want_K) + " x " + std::to_string(want_M) + ", got " +
                             std::to_string(full_K) + " x " + std::to_string(full_M));
  if (row1 < 0) row1 = full_M;
  if (k1 < 0) k1 = full_K;
  const int be = type_block_elems(t.type);
  if (row0 < 0 || row1 > full_M || row0 >= row1 || k0 < 0 || k1 > full_K || k0 >= k1 || k0 % be || k1 % be)
    throw std::runtime_error("tensor '" + t.name + "': shard does not fall on quantization block boundaries");
  m.K = k1 - k0;
  m.M = row1 - row0;
  m.nb = m.K / be;
  const size_t full_row_bytes = t.nbytes / (size_t)full_M;
  const size_t row_bytes = (size_t)m.nb * type_block_bytes(t.type);
  m.bytes = row_bytes * (size_t)m.M;
  const uint8_t* src = t.data + (size_t)row0 * full_row_bytes;
  std::vector<uint8_t> gathered;
  if (m.K != full_K) {   // a K range: the kept blocks of every row, packed
    gathered.resize(m.bytes);
    const size_t off = (size_t)(k0 / be) * type_block_bytes(t.type);
    for (int r = 0; r < m.M; r++) memcpy(gathered.data() + (size_t)r * row_bytes, src + (size_t)r * full_row_bytes + off, row_bytes);
    src = gathered.data();
  }
  int rows_per_chunk = (int)std::max<size_t>(ST_ROWS, UP_CHUNK / row_bytes / ST_ROWS * ST_ROWS);   // whole 16-row tiles
  if (row_bytes * ST_ROWS > UP_CHUNK) throw std::runtime_error("tensor '" + t.name + "': rows too long for the upload staging buffers");
  uint16_t *st = nullptr, *qs = nullptr, *qh = nullptr, *d = nullptr, *mn = nullptr;
  const bool kq = type_is_kquant(m.type);
  if (kq) {
    st = (uint16_t*)alloc(st_matrix_bytes(m.type, m.M, m.nb));
    m.st = (const uint8_t*)st;
  } else {
    const PlaneSizes ps = plane_sizes(m.type, m.M, m.nb, m.bytes);
    qs = (uint16_t*)alloc(ps.qs);
    if (ps.qh) qh = (uint16_t*)alloc(ps.qh);
    if (ps.d) d = (uint16_t*)alloc(ps.d);
    if (ps.mn) mn = (uint16_t*)alloc(ps.mn);
    m.qs = (const uint8_t*)qs; m.qh = (const uint8_t*)qh; m.d = d; m.mn = mn;
  }
  for (int r0 = 0; r0 < m.M; r0 += rows_per_chunk) {
    const int rows = std::min(rows_per_chunk, m.M - r0);
    const size_t n = (size_t)rows * row_bytes;
    const int slot = up.push(src + (size_t)r0 * row_bytes, n);
    if (kq) {
      const size_t sb = st_matrix_bytes(m.type, rows, m.nb);
      const int grid = (int)std::min<size_t>((sb / 2 + 255) / 256, (size_t)sm_count_ * 32);
      k_repack_stream<<<grid, 256, 0, up.st[slot]>>>(m.type, up.dev[slot], rows, m.nb, st + (size_t)(r0 / ST_ROWS) * m.nb * st_block_bytes(m.type) / 2);
    } else {
      const size_t n_u16 = n / 2;
      const size_t blk0 = (size_t)r0 * m.nb;
      const int grid = (int)std::min<size_t>((n_u16 + 255) / 256, (size_t)sm_count_ * 32);
      const bool nib = m.type == GT_Q4_0 || m.type == GT_Q5_0 || m.type == GT_Q4_1 || m.type == GT_Q5_1;   // 16 B of nibbles per block
      uint16_t* qdst = qs + (nib ? blk0 * 8 : (m.type == GT_Q8_0 ? blk0 * 16 : (size_t)r0 * row_bytes / 2));
      k_repack<<<grid, 256, 0, up.st[slot]>>>(m.type, (const uint16_t*)up.dev[slot], n_u16, qdst, qh ? qh + blk0 * 2 : nullptr, d ? d + blk0 : nullptr,
                                              mn ? mn + blk0 : nullptr);
    }
    CTB_CUDA(cudaGetLastError());
    up.finish(slot);
  }
  return m;
}

const float* Engine::upload_vector(const GGUFFile& g, const std::string& name, bool required, int want_n) {
  const GGUFTensor* t = g.tensor(name);
  if (!t) {
    if (required) throw std::runtime_error("tensor '" + name + "' not found");
    return nullptr;
  }
  if (t->type != T_F32) throw std::runtime_error("tensor '" + name + "' must be f32");
  if ((long)t->ne[0] * (long)t->ne[1] != (long)want_n) throw std::runtime_error("tensor '" + name + "' has wrong shape");
  float* d = (float*)alloc(t->nbytes);
  CTB_CUDA(cudaMemcpy(d, t->data, t->nbytes, cudaMemcpyHostToDevice));
  return d;
}

TPShard tp_shard(int n_embd, int n_head, int n_head_kv, int n_ff, int rank, int world) {
  if (world < 1 || rank < 0 || rank >= world || n_head <= 0 || n_head_kv <= 0 || n_embd % n_head || n_head % n_head_kv) throw std::runtime_error("tensor parallel: bad shape or rank");
  const int hd = n_embd / n_head;
  auto gcd = [](int a, int b) { while (b) { const int t = a % b; a = b; b = t; } return a; };
  const int group = 256 / gcd(256, hd);   // query heads per 256-element block of the attention output (2 for head_dim 128)
  if ((hd * group) % 256 || n_head % group || n_ff % 256) throw std::runtime_error("tensor parallel: heads / n_ff do not tile into 256-element blocks");
  auto split = [&](int units, int r0) {   // first element of part r0 when `units` are dealt as evenly as possible (the first units % world parts get one more)
    const int base = units / world, extra = units % world;
    return r0 * base + std::min(r0, extra);
  };
  TPShard s;
  s.rank = rank; s.world = world;
  s.head0 = split(n_head / group, rank) * group; s.head1 = split(n_head / group, rank + 1) * group;
  s.ff0 = split(n_ff / 256, rank) * 256; s.ff1 = split(n_ff / 256, rank + 1) * 256;
  const int per_kv = n_head / n_head_kv;
  s.kv0 = s.head1 > s.head0 ? s.head0 / per_kv : 0;
  s.kv1 = s.head1 > s.head0 ? (s.head1 - 1) / per_kv + 1 : 0;
  return s;
}

Engine::Engine(const HParams& hp, int device, const TPShard& tp) : hp_(hp), tp_(tp), device_(device) {}

// Delegating first makes the engine constructed before init runs, so ~Engine also runs when init throws.
Engine::Engine(const GGUFFile& g, const HParams& hp, int device, const TPShard& tp) : Engine(hp, device, tp) { init(g); }

void Engine::init(const GGUFFile& g) {
  CTB_CUDA(cudaSetDevice(device_));
  cudaDeviceProp prop;
  CTB_CUDA(cudaGetDeviceProperties(&prop, device_));
  sm_count_ = prop.multiProcessorCount;
  // refuse what the kernels cannot run BEFORE the model-sized allocations are made
  for (const auto& t : g.tensors)
    if (t.n_dims >= 2 && !supported_matrix_type(t.type))
      throw std::runtime_error("tensor '" + t.name + "': quantization type " + std::to_string(t.type) + " is not supported by the CUDA path");
  stream_ = Stream(cudaStreamNonBlocking);
  ev0_ = Event(cudaEventDefault);
  ev1_ = Event(cudaEventDefault);

  arena_size_ = engine_arena_bytes(g, hp_);
  arena_ = DevMem(arena_size_);
  const auto t_load0 = std::chrono::steady_clock::now();
  Uploader up;
  up.init((uint8_t*)alloc(UP_CHUNK * UP_BUFS));

  // ---- weights (shapes follow from the hyper-parameters: llama.cpp:1878-1934 llama, 1948-2012 falcon)
  const std::string pfx = "blk.";
  const int n_embd = hp_.n_embd, gqa = hp_.n_embd_gqa(), n_ff = hp_.n_ff;
  nh_ = hp_.n_head; nkv_ = hp_.n_head_kv; nff_ = hp_.n_ff;
  const int hd0 = hp_.head_dim();
  if (tp_.world > 1) {
    const int per_kv = hp_.n_head / hp_.n_head_kv;
    if (hp_.falcon) throw std::runtime_error("tensor parallel mode covers the llama graph only");
    if (!tp_.comm) throw std::runtime_error("tensor parallel mode needs a communicator");
    if (tp_.head1 <= tp_.head0 || tp_.ff1 <= tp_.ff0) throw std::runtime_error("tensor parallel: more ranks than 256-element blocks to share out");
    if (tp_.head0 % per_kv || tp_.head1 % per_kv) throw std::runtime_error("tensor parallel: a rank's query heads must cover whole KV groups");
    nh_ = tp_.head1 - tp_.head0; nkv_ = tp_.kv1 - tp_.kv0; nff_ = tp_.ff1 - tp_.ff0;
    prefill_on_ = false;   // prompts go through the single-token path (the batched kernel has no exchange step)
  }
  const int q0 = tp_.world > 1 ? tp_.head0 * hd0 : 0, q1 = tp_.world > 1 ? tp_.head1 * hd0 : n_embd;        // rows of wq = K range of wo
  const int g0 = tp_.world > 1 ? tp_.kv0 * hd0 : 0, g1 = tp_.world > 1 ? tp_.kv1 * hd0 : gqa;               // rows of wk / wv
  const int f0 = tp_.world > 1 ? tp_.ff0 : 0, f1 = tp_.world > 1 ? tp_.ff1 : n_ff;                          // rows of w1 / w3 = K range of w2
  {
    const GGUFTensor& te = g.need_tensor("token_embd.weight");
    if (!supported_matrix_type(te.type)) throw std::runtime_error("token_embd.weight: unsupported type");
    if ((int)te.ne[0] != n_embd || (long)(te.ne[1] * te.ne[2] * te.ne[3]) != (long)hp_.n_vocab) throw std::runtime_error("token_embd.weight has wrong shape");
    uint8_t* d = (uint8_t*)alloc(te.nbytes);
    CTB_CUDA(cudaMemcpy(d, te.data, te.nbytes, cudaMemcpyHostToDevice));
    tok_embd_ = d; tok_type_ = (int)te.type;
    tok_row_bytes_ = te.ne[0] / type_block_elems(te.type) * type_block_bytes(te.type);
  }
  out_norm_ = upload_vector(g, "output_norm.weight", true, n_embd);
  out_norm_b_ = upload_vector(g, "output_norm.bias", hp_.falcon, n_embd);
  output_ = upload_matrix(g.need_tensor("output.weight"), up, n_embd, hp_.n_vocab);
  size_t wbytes = output_.bytes;
  layers_.resize(hp_.n_layer);
  for (int il = 0; il < hp_.n_layer; il++) {
    LayerW& L = layers_[il];
    const std::string b = pfx + std::to_string(il) + ".";
    L.attn_norm = upload_vector(g, b + "attn_norm.weight", true, n_embd);
    if (hp_.falcon) {
      L.attn_norm_b = upload_vector(g, b + "attn_norm.bias", true, n_embd);
      L.attn_norm2 = upload_vector(g, b + "attn_norm_2.weight", false, n_embd);
      if (L.attn_norm2) L.attn_norm2_b = upload_vector(g, b + "attn_norm_2.bias", true, n_embd);
      L.wqkv = upload_matrix(g.need_tensor(b + "attn_qkv.weight"), up, n_embd, n_embd + 2 * gqa);
      L.wo = upload_matrix(g.need_tensor(b + "attn_output.weight"), up, n_embd, n_embd);
      L.w3 = upload_matrix(g.need_tensor(b + "ffn_up.weight"), up, n_embd, n_ff);
      L.w2 = upload_matrix(g.need_tensor(b + "ffn_down.weight"), up, n_ff, n_embd);
      wbytes += L.wqkv.bytes + L.wo.bytes + L.w3.bytes + L.w2.bytes;
    } else {
      L.ffn_norm = upload_vector(g, b + "ffn_norm.weight", true, n_embd);
      L.wq = upload_matrix(g.need_tensor(b + "attn_q.weight"), up, n_embd, n_embd, q0, q1);
      L.wk = upload_matrix(g.need_tensor(b + "attn_k.weight"), up, n_embd, gqa, g0, g1);
      L.wv = upload_matrix(g.need_tensor(b + "attn_v.weight"), up, n_embd, gqa, g0, g1);
      L.wo = upload_matrix(g.need_tensor(b + "attn_output.weight"), up, n_embd, n_embd, 0, -1, q0, q1);
      L.w1 = upload_matrix(g.need_tensor(b + "ffn_gate.weight"), up, n_embd, n_ff, f0, f1);
      L.w2 = upload_matrix(g.need_tensor(b + "ffn_down.weight"), up, n_ff, n_embd, 0, -1, f0, f1);
      L.w3 = upload_matrix(g.need_tensor(b + "ffn_up.weight"), up, n_embd, n_ff, f0, f1);
      wbytes += L.wq.bytes + L.wk.bytes + L.wv.bytes + L.wo.bytes + L.w1.bytes + L.w2.bytes + L.w3.bytes;
      if (act_format_for(L.w1.type) != act_format_for(L.w3.type)) throw std::runtime_error("ffn_gate / ffn_up use incompatible quantization families");
    }
  }
  stats.weight_bytes_per_token = wbytes;
  up.drain();
  stats.load_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_load0).count();
  stats.load_bytes = up.bytes;

  // ---- lookup tables, built with the host libm exactly like ggml_init does (ggml.c:4319-4333)
  {
    const HostTables t = host_tables();
    silu_tab_ = (uint16_t*)alloc(65536 * 2); gelu_tab_ = (uint16_t*)alloc(65536 * 2); exp_tab_ = (uint16_t*)alloc(65536 * 2);
    CTB_CUDA(cudaMemcpy(silu_tab_, t.silu.data(), 65536 * 2, cudaMemcpyHostToDevice));
    CTB_CUDA(cudaMemcpy(gelu_tab_, t.gelu.data(), 65536 * 2, cudaMemcpyHostToDevice));
    CTB_CUDA(cudaMemcpy(exp_tab_, t.ex.data(), 65536 * 2, cudaMemcpyHostToDevice));
  }
  // ---- RoPE table: same recurrence, same libm calls as ggml.c:12482-12529
  {
    const std::vector<float2> tab = rope_table(hp_.n_ctx, hp_.head_dim(), hp_.n_rot, hp_.rope_base, hp_.rope_scale);
    rope_ = (float2*)alloc(tab.size() * sizeof(float2));
    CTB_CUDA(cudaMemcpy(rope_, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice));
  }
  // ---- KV cache + workspace
  const size_t gqa_l = (size_t)nkv_ * hp_.head_dim(), qw_l = (size_t)nh_ * hp_.head_dim();   // this rank's K/V and Q widths
  const size_t kv = (size_t)hp_.n_layer * hp_.n_ctx * nkv_ * k_stride(hp_.head_dim());   // K rows padded to 8 halves (attention.cuh)
  const size_t vv = (size_t)hp_.n_layer * kv_ctx_pad(hp_.n_ctx) * gqa_l;
  kc_ = (uint16_t*)alloc(kv * 2 * hp_.n_seq);   // [slot][layer]...: slot 0 is the single-sequence cache
  vc_ = (uint16_t*)alloc(vv * 2 * hp_.n_seq);
  CTB_CUDA(cudaMemset(kc_, 0, kv * 2 * hp_.n_seq));
  CTB_CUDA(cudaMemset(vc_, 0, vv * 2 * hp_.n_seq));
  const size_t qkv = qw_l + 2 * gqa_l;
  d_state_ = (int*)alloc(64);
  xa_ = (float*)alloc(hp_.n_embd * 4); xb_ = (float*)alloc(hp_.n_embd * 4);
  qkv_ = (float*)alloc(qkv * 4);
  attn_ = (float*)alloc(hp_.n_embd * 4); attn_o_ = (float*)alloc(hp_.n_embd * 4);
  ffn_ = (float*)alloc((size_t)nff_ * 4);
  ffn2_ = (float*)alloc((size_t)nff_ * 4);
  d_logits_ = (float*)alloc((size_t)hp_.n_vocab * 4);
  d_embd_ = (float*)alloc(hp_.n_embd * 4);
  {
    const size_t nl = (size_t)hp_.n_seq * hp_.n_vocab, ne = (size_t)hp_.n_seq * hp_.n_embd, bytes = (nl + ne) * 4 + (size_t)hp_.n_seq * 8;
    kept_logits_ = (float*)alloc(bytes);
    kept_embd_ = kept_logits_ + nl;
    kept_pick_ = (int*)(kept_embd_ + ne);
    CTB_CUDA(cudaMemset(kept_logits_, 0, bytes));
  }
  d_sync_ = (unsigned*)alloc(64);
  CTB_CUDA(cudaMemset(d_state_, 0, 64));
  CTB_CUDA(cudaMemset(d_sync_, 0, 64));
  h_logits_ = HostMem((size_t)hp_.n_vocab * 4);
  h_embd_ = HostMem((size_t)hp_.n_embd * 4);
  memset(h_logits_.get(), 0, (size_t)hp_.n_vocab * 4);
  memset(h_embd_.get(), 0, (size_t)hp_.n_embd * 4);
  step_ring_ = StateRing(d_state_, 4, 512);

  if (const char* e = getenv("CTB_NO_PDL")) pdl_ = !(e[0] == '1');
  if (const char* e = getenv("CTB_NO_SPEC")) spec_on_ = !(e[0] == '1');
  if (const char* e = getenv("CTB_STEP_FUSE")) fused_ = !(e[0] == '0');
  if (const char* e = getenv("CTB_NO_PREFILL")) prefill_on_ = !(e[0] == '1');
  if (const char* e = getenv("CTB_PREFILL_MIN")) prefill_min_ = std::max(1, atoi(e));
  h_spec_tok_ = HostMem(16);
  {   // the kernels' watchdog words: host memory the device can write and the host can read after a trapped launch
    h_dbg_ = HostMem(64, true);
    memset(h_dbg_.get(), 0, 64);
    int* d = nullptr;
    CTB_CUDA(cudaHostGetDevicePointer(&d, h_dbg_.get(), 0));
    CTB_CUDA(st_set_debug_words(d));
    g_watchdog_words = h_dbg_.as<int>();
  }
  ev_pick_ = Event(cudaEventDisableTiming);
  ev_sample_ = Event(cudaEventDisableTiming);
  CTB_CUDA(matvec_set_smem_limit(MV_SMEM_LIMIT));
  CTB_CUDA(cudaFuncSetAttribute(attn_kernel(hp_.head_dim()), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attn_smem_bytes(hp_.n_ctx, hp_.head_dim())));
  if (tp_.world > 1) tp_setup_peer();
  build_ops();
  if (tp_peer_)
    for (const StepOp& op : ops_)
      if (op.ph.kind == PH_MATVEC && !op.stream) throw std::runtime_error("tensor parallel (fused exchange): every mat-vec must run in the step kernel (K-quant weights)");
  CTB_CUDA(cudaDeviceSynchronize());
  build_graphs();
}

Engine::~Engine() {
  cudaSetDevice(device_);   // the members free on the engine's device, behind its work
  cudaDeviceSynchronize();
  for (int r = 0; r < 8; r++)
    if (xc_ll_[r] && r != tp_.rank) cudaIpcCloseMemHandle(xc_ll_[r]);
  if (xc_region_) cudaFree(xc_region_);
}

void Engine::set_stream(cudaStream_t s) { stream_.set_stream(s); }

static MVSeg seg(const DevMat& w, float* out, int epi = EPI_STORE, const float* res = nullptr, const float* res2 = nullptr) {
  MVSeg s;
  s.w = w; s.out = out; s.res = res; s.res2 = res2; s.epi = epi;
  return s;
}

// The op list of one token through the whole model (the reference rebuilds this graph on every eval, llama.cpp:2872-2876;
// here it is a static schedule whose pointers never change): EMBED, per layer {QKV mat-vec(s), ATTN, WO, UP, DOWN}, then the
// HEAD mat-vec and the greedy PICK.  {token, n_past} are read from d_state_ on the device.
void Engine::push_matvec(MVParams& p, int kind) {
  p.silu_tab = silu_tab_;
  p.gelu_tab = gelu_tab_;
  StepOp op{};
  op.ph = step_supports(p) ? matvec_phase(p) : Phase{};
  op.ph.kind = PH_MATVEC;
  op.ph.mv = p;
  op.mvk = kind;
  op.stream = step_supports(p);
  if (op.stream) op.ph.mv.act = ACT_Q8_K;
  ops_.push_back(op);
}

void Engine::tp_all_reduce(float* buf, int n, cudaStream_t st) {
  const NcclApi& nccl = NcclApi::get();
  nccl.check(nccl.AllReduce(buf, buf, (size_t)n, ncclFloat, ncclSum, (ncclComm_t)tp_.comm, st), "all-reduce");
}

// Fused exchange set-up: allocate this rank's region, hand its CUDA IPC handle to the peers (the NCCL communicator carries the 64
// bytes), map theirs.  All-or-nothing across ranks: if any rank cannot map a peer, every rank stays on the NCCL all-reduce path.
void Engine::tp_setup_peer() {
  const NcclApi& nccl = NcclApi::get();
  const int W = tp_.world;
  const size_t bytes = align_up((size_t)2 * W * hp_.n_embd * sizeof(uint2), 256);
  int ok = 1;
  cudaIpcMemHandle_t mine;
  std::vector<cudaIpcMemHandle_t> all(W);
  uint8_t* d_h = (uint8_t*)alloc(sizeof(cudaIpcMemHandle_t) * W + 16, 256);
  int* d_ok = (int*)(d_h + sizeof(cudaIpcMemHandle_t) * W);
  if (W > XC_MAX_WORLD || getenv("CTB_TP_NCCL")) ok = 0;
  if (ok && cudaMalloc(&xc_region_, bytes) != cudaSuccess) { xc_region_ = nullptr; ok = 0; }
  if (ok) {
    CTB_CUDA(cudaMemset(xc_region_, 0, bytes));
    if (cudaIpcGetMemHandle(&mine, xc_region_) != cudaSuccess) ok = 0;
  }
  if (!ok) memset(&mine, 0, sizeof(mine));
  cudaGetLastError();
  CTB_CUDA(cudaMemcpy(d_h + sizeof(mine) * tp_.rank, &mine, sizeof(mine), cudaMemcpyHostToDevice));
  nccl.check(nccl.AllGather(d_h + sizeof(mine) * tp_.rank, d_h, sizeof(mine), ncclChar, (ncclComm_t)tp_.comm, stream_), "all-gather of the IPC handles");
  CTB_CUDA(cudaStreamSynchronize(stream_));
  CTB_CUDA(cudaMemcpy(all.data(), d_h, sizeof(mine) * W, cudaMemcpyDeviceToHost));
  for (int r = 0; r < W && ok; r++) {
    void* base = xc_region_;
    if (r != tp_.rank && cudaIpcOpenMemHandle(&base, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); break; }
    xc_ll_[r] = (uint2*)base;
  }
  CTB_CUDA(cudaMemcpy(d_ok, &ok, 4, cudaMemcpyHostToDevice));
  nccl.check(nccl.AllReduce(d_ok, d_ok, 1, ncclInt, ncclMin, (ncclComm_t)tp_.comm, stream_), "all-reduce");
  CTB_CUDA(cudaStreamSynchronize(stream_));
  CTB_CUDA(cudaMemcpy(&ok, d_ok, 4, cudaMemcpyDeviceToHost));
  tp_peer_ = ok != 0;
  if (!tp_peer_ && tp_.rank == 0 && !getenv("CTB_TP_NCCL"))
    fprintf(stderr, "ctransformers-b200: peer memory between the ranks is not available; the tensor-parallel exchange uses NCCL all-reduce\n");
}

void Engine::build_ops() {
  // nh_ / nkv_ / nff_ are this rank's share (the whole model without tensor parallelism)
  const int n_embd = hp_.n_embd, hd = hp_.head_dim(), n_kv = nkv_, gqa = nkv_ * hp_.head_dim(), qw = nh_ * hp_.head_dim();
  const bool tp = tp_.world > 1;
  const bool tp_lead = tp_.rank == 0;   // the rank whose partial sum carries the residual
  int n_xchg = 0;                       // exchanges so far in the program
  bool xchg_due = false;                // fused mode: the next mat-vec phase consumes the exchange the last one produced
  float* x_sum_into = nullptr;
  auto fill_xc = [&](XchgParams& xc, int role) {
    xc.world = tp_.world; xc.rank = tp_.rank; xc.index = n_xchg; xc.n = n_embd; xc.role = role;
    for (int r = 0; r < tp_.world; r++) xc.ll[r] = xc_ll_[r];
  };
  auto push_xchg = [&](float* buf) {    // all-reduce of a row-parallel mat-vec's partial sums (+ the residual, once)
    if (tp_peer_) {                     // fused: that phase's epilogue sends its rows to every rank; the next phase sums them into buf
      fill_xc(ops_.back().ph.xc, 2);
      xchg_due = true;
      x_sum_into = buf;
      return;
    }
    StepOp op{};
    op.ph.kind = PH_XCHG;
    op.ph.em.out = buf; op.ph.em.K = n_embd;
    ops_.push_back(op);
  };
  auto take_input = [&](MVParams& p) {   // fused: the input is the sum of the ranks' vectors of the exchange that is due
    if (!xchg_due) return;
    p.x = (const float*)xc_ll_[tp_.rank]; p.x_mode = 2; p.x_parts = tp_.world; p.x_stride = n_embd; p.sum_out = x_sum_into;
  };
  auto mark_exchange = [&](size_t first_op) {
    if (!xchg_due) return;
    if (ops_.size() != first_op + 1) throw std::runtime_error("tensor parallel (fused exchange): the consumer of an exchange must be one mat-vec phase");
    fill_xc(ops_[first_op].ph.xc, 1);
    n_xchg++;
    xchg_due = false; x_sum_into = nullptr;
  };
  const float kq_scale = 1.0f / sqrtf((float)n_embd / (float)hp_.n_head);
  ops_.clear();
  {
    StepOp op{};
    op.ph.kind = PH_EMBED;
    op.ph.em.table = tok_embd_; op.ph.em.row_bytes = tok_row_bytes_; op.ph.em.tokens = d_state_; op.ph.em.out = xa_;
    op.ph.em.type = tok_type_; op.ph.em.K = n_embd; op.ph.em.n_vocab = hp_.n_vocab;
    ops_.push_back(op);
  }
  float* x = xa_;
  float* y = xb_;
  for (int il = 0; il < hp_.n_layer; il++) {
    const LayerW& L = layers_[il];
    uint16_t* kc = kc_ + (size_t)il * hp_.n_ctx * n_kv * k_stride(hd);
    uint16_t* vc = vc_ + (size_t)il * gqa * kv_ctx_pad(hp_.n_ctx);
    AttnParams ap{};
    ap.kc = kc; ap.vc = vc; ap.out = attn_; ap.exp_tab = exp_tab_; ap.state = d_state_; ap.kq_scale = kq_scale;
    ap.n_head = nh_; ap.n_kv = n_kv; ap.hd = hd; ap.n_ctx = hp_.n_ctx; ap.rope = rope_; ap.neox = hp_.falcon ? 1 : 0;
    auto push_attn = [&]() {
      StepOp op{};
      op.ph.kind = PH_ATTN;
      op.ph.at = ap;
      ops_.push_back(op);
    };

    if (!hp_.falcon) {
      float* q = qkv_; float* k = qkv_ + qw; float* v = qkv_ + qw + gqa;
      {  // attention_norm + wq/wk/wv
        MVParams p{};
        p.x = x; p.norm_w = L.attn_norm; p.norm_mode = NORM_RMS; p.eps = hp_.eps; p.K = n_embd;
        const size_t first_op = ops_.size();
        take_input(p);
        const DevMat* ws[3] = {&L.wq, &L.wk, &L.wv};
        float* outs[3] = {q, k, v};
        bool done[3] = {false, false, false};
        ap.q = q; ap.k = k; ap.v = v; ap.q_stride = qw; ap.kv_stride = gqa;
        for (int i = 0; i < 3; i++) {   // group tensors that share an activation format into one launch
          if (done[i]) continue;
          p.act = act_format_for(ws[i]->type); p.nseg = 0;
          for (int j = i; j < 3; j++)
            if (!done[j] && act_format_for(ws[j]->type) == p.act) { p.seg[p.nseg++] = seg(*ws[j], outs[j]); done[j] = true; }
          push_matvec(p, MVK_QKV);
        }
        mark_exchange(first_op);
      }
      push_attn();
      {  // wo + residual
        MVParams p{};
        p.x = attn_; p.norm_mode = NORM_NONE; p.K = qw; p.act = act_format_for(L.wo.type); p.nseg = 1;
        p.seg[0] = (!tp || tp_lead) ? seg(L.wo, y, EPI_ADD, x) : seg(L.wo, y);
        push_matvec(p, MVK_WO);
        if (tp) push_xchg(y);
      }
      {  // ffn_norm + gate and up projections as two independent row sets: silu(gate) is stored, the product with up is formed
         // where ffn_down stages its input
        MVParams p{};
        p.x = y; p.norm_w = L.ffn_norm; p.norm_mode = NORM_RMS; p.eps = hp_.eps; p.K = n_embd;
        const size_t first_op = ops_.size();
        take_input(p);
        p.act = act_format_for(L.w1.type); p.nseg = 2;
        p.seg[0] = seg(L.w1, ffn_, EPI_SILU); p.seg[1] = seg(L.w3, ffn2_);
        push_matvec(p, MVK_UP);
        mark_exchange(first_op);
      }
      {  // w2 on silu(gate)*up, + residual
        MVParams p{};
        p.x = ffn_; p.x2 = ffn2_; p.x_mode = 1; p.norm_mode = NORM_NONE; p.K = nff_; p.act = act_format_for(L.w2.type); p.nseg = 1;
        p.seg[0] = (!tp || tp_lead) ? seg(L.w2, x, EPI_ADD, y) : seg(L.w2, x);
        push_matvec(p, MVK_DOWN);
        if (tp) push_xchg(x);
      }
      // x now holds the next layer's input
    } else {
      const int qkv_w = (hp_.n_head + 2 * n_kv) * hd;
      float* q = qkv_; float* k = qkv_ + (size_t)hp_.n_head * hd; float* v = k + (size_t)n_kv * hd;
      const bool two_norms = L.attn_norm2 != nullptr;
      const bool fuse = !two_norms && act_format_for(L.wqkv.type) == act_format_for(L.w3.type);
      {  // LayerNorm + wqkv (+ ffn_up → GELU when it shares the normed input)
        MVParams p{};
        p.x = x; p.norm_mode = NORM_LAYER; p.eps = hp_.eps; p.K = n_embd;
        p.norm_w = two_norms ? L.attn_norm2 : L.attn_norm; p.norm_b = two_norms ? L.attn_norm2_b : L.attn_norm_b;
        p.act = act_format_for(L.wqkv.type); p.nseg = 1;
        p.seg[0] = seg(L.wqkv, qkv_);
        if (fuse) { p.seg[1] = seg(L.w3, ffn_, EPI_GELU); p.nseg = 2; }
        ap.q = q; ap.k = k; ap.v = v; ap.q_stride = qkv_w; ap.kv_stride = qkv_w;
        push_matvec(p, MVK_QKV);
      }
      if (!fuse) {
        MVParams p{};
        p.x = x; p.norm_mode = NORM_LAYER; p.eps = hp_.eps; p.K = n_embd; p.norm_w = L.attn_norm; p.norm_b = L.attn_norm_b;
        p.act = act_format_for(L.w3.type); p.nseg = 1;
        p.seg[0] = seg(L.w3, ffn_, EPI_GELU);
        push_matvec(p, MVK_UP);
      }
      push_attn();
      {  // attention output projection
        MVParams p{};
        p.x = attn_; p.norm_mode = NORM_NONE; p.K = n_embd; p.act = act_format_for(L.wo.type); p.nseg = 1;
        p.seg[0] = seg(L.wo, attn_o_);
        push_matvec(p, MVK_WO);
      }
      {  // ffn_down, then + attn_out, then + layer input (llama.cpp:2767-2771 order)
        MVParams p{};
        p.x = ffn_; p.norm_mode = NORM_NONE; p.K = hp_.n_ff; p.act = act_format_for(L.w2.type); p.nseg = 1;
        p.seg[0] = seg(L.w2, y, EPI_ADD2, attn_o_, x);
        push_matvec(p, MVK_DOWN);
      }
      std::swap(x, y);
    }
  }
  n_body_ = (int)ops_.size();
  {
    MVParams p{};
    p.x = x; p.norm_w = out_norm_; p.norm_b = out_norm_b_; p.norm_mode = hp_.falcon ? NORM_LAYER : NORM_RMS; p.eps = hp_.eps; p.K = n_embd;
    const size_t first_op = ops_.size();
    take_input(p);
    p.norm_out = d_embd_; p.act = act_format_for(output_.type); p.nseg = 1;
    p.seg[0] = seg(output_, d_logits_);
    push_matvec(p, MVK_OUT);
    mark_exchange(first_op);

  }
  {
    StepOp op{};
    op.ph.kind = PH_PICK;
    op.ph.pk.logits = d_logits_; op.ph.pk.state = d_state_; op.ph.pk.out_tokens = nullptr; op.ph.pk.n = hp_.n_vocab;   // out_tokens: set in build_graphs
    ops_.push_back(op);
  }
  // ---- the step kernel's shared-memory shape: ring slots fill what the largest activation image leaves
  bool any_stream = false;
  for (const StepOp& op : ops_) any_stream |= op.ph.kind == PH_MATVEC && op.stream;
  std::vector<Phase> phs;
  for (const StepOp& op : ops_) if (op.ph.kind != PH_XCHG && (op.ph.kind != PH_MATVEC || op.stream)) phs.push_back(op.ph);
  const StepLaunch sl = step_launch_plan(phs.data(), (int)phs.size(), sm_count_);
  step_grid_ = sl.grid; step_slots_ = sl.n_slots; step_smem_ = sl.smem; step_q3_ = sl.q3;
  if (const char* e = getenv("CTB_ST_SLOTS")) {   // A/B knob: fewer ring slots = less prefetch in flight
    const int want = atoi(e);
    if (want >= ST_W && want < step_slots_ && want % ST_W == 0) { step_smem_ -= (size_t)(step_slots_ - want) * ST_SLOT; step_slots_ = want; }
  }
  ring_attn_ = st_attn_ring_ok(hp_.n_ctx, step_slots_) && !getenv("CTB_NO_RING_ATTN");
  for (StepOp& op : ops_) if (op.ph.kind == PH_ATTN) op.ph.q6 = ring_attn_ ? 1 : 0;
  if (any_stream && step_slots_ < ST_W) throw std::runtime_error("model rows are too long for the step kernel's shared memory");
  if (any_stream) {
    CTB_CUDA(step_set_smem_limit(step_smem_));
    StepLaunch pl = sl;
    pl.n_slots = step_slots_; pl.smem = step_smem_;
    step_pair_ = step_pair_choose(pl, phs.data(), (int)phs.size());
  } else {
    fused_ = false;
  }
  d_prog_ = (Phase*)alloc((ops_.size() + 1) * sizeof(Phase), 256);
  d_prog_mv_ = (Phase*)alloc((ops_.size() + 1) * sizeof(Phase), 256);
  d_bounds_ = (int*)alloc((ops_.size() + 1) * (size_t)(sm_count_ + 1) * 4, 256);      // per-CTA tile ranges, one row per phase
  d_bounds_mv_ = (int*)alloc((ops_.size() + 1) * (size_t)(sm_count_ + 1) * 4, 256);
}

void Engine::upload_prog(Phase* dst, int* dst_bounds, const std::vector<StepOp>& ops) {
  std::vector<Phase> phs(ops.size());
  for (size_t i = 0; i < ops.size(); i++) phs[i] = ops[i].ph;
  CTB_CUDA(cudaMemcpy(dst, phs.data(), phs.size() * sizeof(Phase), cudaMemcpyHostToDevice));
  std::vector<Phase> run = phs;
  for (size_t i = 0; i < ops.size(); i++) if (ops[i].ph.kind == PH_XCHG || (ops[i].ph.kind == PH_MATVEC && !ops[i].stream)) run[i].kind = -1;   // not a step-kernel phase
  const std::vector<int> b = step_bounds(run.data(), (int)run.size(), sm_count_);
  CTB_CUDA(cudaMemcpy(dst_bounds, b.data(), b.size() * 4, cudaMemcpyHostToDevice));
}

struct ProfMark {
  Event ev;
  int kind;   // the class (profile_step) of the kernel that ends here, or -1 where one starts
};

// Enqueue ops[0, n) on st; returns the kernels launched.  Fused mode: maximal runs of ops the step kernel can take become ONE
// k_step launch (a K-quant model: the whole token); anything else (Q4_0 / Q8_0 / F16 / F32 mat-vecs) runs as its own kernel.
// Un-fused mode (CTB_STEP_FUSE=0): one kernel per op, K-quant mat-vecs as one-phase k_step launches.  marks: an event before and
// after every kernel.
long Engine::enqueue_ops(const std::vector<StepOp>& ops, const Phase* d_prog, const int* d_bounds, int n, cudaStream_t st, bool fused,
                         std::vector<ProfMark>* marks) {
  long launches = 0;
  auto mark = [&](int kind) {
    if (!marks) return;
    marks->push_back({Event(cudaEventDefault), kind});
    CTB_CUDA(cudaEventRecord(marks->back().ev, st));
  };
  StepLaunch step_shape_;
  step_shape_.grid = step_grid_; step_shape_.n_slots = step_slots_; step_shape_.smem = step_smem_; step_shape_.gen = !attn_fast_hd(hp_.head_dim());
  step_shape_.q3 = step_q3_;
  step_shape_.pair = step_pair_;
  auto capable = [&](const StepOp& op) { return op.ph.kind != PH_XCHG && (op.ph.kind != PH_MATVEC || op.stream); };
  int i = 0;
  while (i < n) {
    const StepOp& op = ops[i];
    if (fused && capable(op)) {
      int j = i;
      while (j < n && capable(ops[j])) j++;
      mark(-1);
      CTB_CUDA(launch_step(step_shape_, st, d_prog + i, d_bounds + (size_t)i * (sm_count_ + 1), j - i, d_sync_, false, nullptr, tp_peer_));
      launches++;
      mark(0);
      i = j;
      continue;
    }
    mark(-1);
    switch (op.ph.kind) {
      case PH_EMBED:
        k_embed<<<1, 256, 0, st>>>(op.ph.em);
        launches++;
        mark(3);
        break;
      case PH_ATTN:
        CTB_CUDA(launch_kernel(attn_kernel(hp_.head_dim()), dim3(nh_, 1, attn_groups(hp_.head_dim())), dim3(ATTN_THREADS), attn_smem_bytes(hp_.n_ctx, hp_.head_dim()), st, pdl_, op.ph.at));
        launches++;
        mark(1);
        break;
      case PH_XCHG:
        tp_all_reduce(op.ph.em.out, op.ph.em.K, st);
        mark(3);
        break;
      case PH_PICK:
        k_argmax<<<1, ARGMAX_THREADS, 0, st>>>(d_logits_, hp_.n_vocab, d_state_ + 4);
        k_advance<<<1, 1, 0, st>>>(d_state_, d_tokens_out_.as<int>());
        launches += 2;
        mark(3);
        break;
      default:
        if (op.stream) {
          CTB_CUDA(launch_step(step_shape_, st, d_prog + i, d_bounds + (size_t)i * (sm_count_ + 1), 1, d_sync_));
        } else {
          const MVLaunch L = matvec_launch_shape(op.ph.mv, sm_count_);
          CTB_CUDA(launch_matvec_kernel(L, st, op.ph.mv, pdl_));
        }
        launches++;
        mark(0);
    }
    i++;
  }
  CTB_CUDA(cudaGetLastError());
  return launches;
}

// One eager decode step, one kernel per op (un-fused), a CUDA event around every kernel: the kernel classes' share of a step.
int Engine::profile_step(int token, int n_past, double ms_by_kind[4], int count_by_kind[4]) {
  DeviceGuard dev_guard(device_);
  if (tp_.world > 1) throw std::runtime_error("not available in tensor-parallel mode (every rank must run the same launches)");
  drop_lookahead();
  put_step(token, n_past, n_past + 1);
  std::vector<ProfMark> marks;
  enqueue_ops(ops_, d_prog_, d_bounds_, n_body_ + 1, stream_, false, &marks);
  CTB_CUDA(cudaStreamSynchronize(stream_));
  int n = 0;
  for (size_t i = 1; i < marks.size(); i++) {
    float ms = 0;
    cudaEventElapsedTime(&ms, marks[i - 1].ev, marks[i].ev);
    const int k = marks[i].kind;
    if (k >= 0 && k < 4) { ms_by_kind[k] += ms; count_by_kind[k]++; n++; }
  }
  return n;
}

// The step's mat-vec phases alone (same kernel, same parameters, same order; no attention / embedding / pick), replayed as a
// CUDA graph: their duration under in-step conditions is what bench.py's roofline for the mat-vec uses.  mask: bit k set =
// keep the mat-vecs of kind k (0 = all).  with_attn: keep the attention phases too (times the dependency chain as it is).
double Engine::time_matvec_only(int reps, long* launches, unsigned mask) {
  if (!mask) mask = ~0u;
  if (tp_.world > 1) throw std::runtime_error("not available in tensor-parallel mode (every rank must run the same launches)");
  drop_lookahead();
  DeviceGuard dev_guard(device_);
  std::vector<StepOp> sel;
  for (int i = 0; i <= n_body_; i++)
    if (ops_[i].ph.kind == PH_MATVEC && ((mask >> ops_[i].mvk) & 1)) sel.push_back(ops_[i]);
  if (sel.empty()) { if (launches) *launches = 0; return 0.0; }
  upload_prog(d_prog_mv_, d_bounds_mv_, sel);
  GraphExec ex;
  {
    const Stream cap(cudaStreamNonBlocking);
    cudaGraph_t g;
    CTB_CUDA(cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal));
    enqueue_ops(sel, d_prog_mv_, d_bounds_mv_, (int)sel.size(), cap, fused_);
    CTB_CUDA(cudaStreamEndCapture(cap, &g));
    ex = GraphExec(g);
    cudaGraphDestroy(g);
  }
  if (launches) *launches = (long)sel.size();
  const Event e0(cudaEventDefault), e1(cudaEventDefault);
  for (int i = 0; i < 3; i++) CTB_CUDA(cudaGraphLaunch(ex, stream_));
  CTB_CUDA(cudaEventRecord(e0, stream_));
  for (int i = 0; i < reps; i++) CTB_CUDA(cudaGraphLaunch(ex, stream_));
  CTB_CUDA(cudaEventRecord(e1, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  return (double)ms / reps;
}

// One fused decode step with the step kernel stamping %globaltimer per phase and CTA (4 stamps: barrier passed, input staged,
// first weight item ready, phase done + 4 stamps of the grid barrier in front of the phase).  out: n_phases x {kind, mvk} then n_phases x n_cta x 8 stamps; returns n_phases or -(words needed).
long Engine::trace_step(int token, int n_past, unsigned long long* out, long cap_words) {
  DeviceGuard dev_guard(device_);
  if (tp_.world > 1) throw std::runtime_error("not available in tensor-parallel mode (every rank must run the same launches)");
  drop_lookahead();
  const int n = n_body_ + 1;
  for (int i = 0; i < n; i++)
    if (ops_[i].ph.kind == PH_MATVEC && !ops_[i].stream) return 0;
  const long need = 2L * n + 8L * n * step_grid_;
  if (need > cap_words) return -need;
  const DevMem buf((size_t)n * step_grid_ * 64);
  CTB_CUDA(cudaMemset(buf.get(), 0, (size_t)n * step_grid_ * 64));
  StepLaunch L;
  L.grid = step_grid_; L.n_slots = step_slots_; L.smem = step_smem_; L.gen = !attn_fast_hd(hp_.head_dim()); L.q3 = step_q3_; L.pair = step_pair_;
  for (int rep = 0; rep < 3; rep++) {   // the last (warm) run is the one read back
    put_step(token, n_past, n_past + 1);
    CTB_CUDA(launch_step(L, stream_, d_prog_, d_bounds_, n, d_sync_, false, buf.as<unsigned long long>()));
    CTB_CUDA(cudaStreamSynchronize(stream_));
  }
  for (int i = 0; i < n; i++) { out[2 * i] = (unsigned long long)ops_[i].ph.kind; out[2 * i + 1] = (unsigned long long)ops_[i].mvk; }
  CTB_CUDA(cudaMemcpy(out + 2 * n, buf.get(), (size_t)n * step_grid_ * 64, cudaMemcpyDeviceToHost));
  return n;
}

void Engine::build_graphs() {
  tokens_out_cap_ = std::max(hp_.n_ctx, 4096);
  d_tokens_out_ = DevMem((size_t)tokens_out_cap_ * 4);
  h_tokens_out_ = HostMem((size_t)tokens_out_cap_ * 4);
  const Stream cap(cudaStreamNonBlocking);
  ops_.back().ph.pk.out_tokens = d_tokens_out_.as<int>();
  upload_prog(d_prog_, d_bounds_, ops_);
  long launches = 0;
  auto capture = [&](bool logits, bool greedy) {
    cudaGraph_t g;
    CTB_CUDA(cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal));
    // (fused tensor-parallel exchange: the head phase consumes the last layer's exchange, so every program contains it)
    launches = enqueue_ops(ops_, d_prog_, d_bounds_, n_body_ + (logits || tp_peer_ ? 1 : 0) + (greedy ? 1 : 0), cap, fused_);
    CTB_CUDA(cudaStreamEndCapture(cap, &g));
    GraphExec ex(g);
    cudaGraphDestroy(g);
    return ex;
  };
  graph_nolog_ = capture(false, false);
  graph_greedy_ = capture(true, true);
  graph_full_ = capture(true, false);
  stats.launches = launches;
}

// After an eval: pick the greedy next token on the device and — once the caller has proven to decode greedily (its last
// tokens were exactly those picks) — run the step for that token right away, while the host is still sampling and crossing
// the FFI.  The next eval() that asks for exactly this token at this position only has to fetch the result; any other request
// simply runs after it (stream order) and overwrites the same KV slot, so a wrong guess costs time, never correctness.
void Engine::after_eval(int next_pos) {
  spec_pending_ = false;
  spec_deferred_ = false;
  spec_pos_ = -1;
  // the look-ahead step writes K/V slot next_pos: only when nothing valid can live there (append-only decoding).  A caller
  // that re-evaluates an earlier position and later continues past it keeps its cache contents.
  if (!spec_on_ || next_pos >= hp_.n_ctx || next_pos < kv_high_) return;
  k_argmax<<<1, ARGMAX_THREADS, 0, stream_>>>(d_logits_, hp_.n_vocab, d_state_ + 4);
  k_advance<<<1, 1, 0, stream_>>>(d_state_, d_tokens_out_.as<int>());
  CTB_CUDA(cudaMemcpyAsync(h_spec_tok_.get(), d_state_ + 4, 8, cudaMemcpyDeviceToHost, stream_));   // {greedy pick, how many logits equal the maximum}
  CTB_CUDA(cudaEventRecord(ev_pick_, stream_));
  spec_pos_ = next_pos;
  if (spec_streak_ >= 2) {
    // The persistent step kernel fills every SM, so whatever is enqueued behind the look-ahead step waits for all of it.  A
    // caller whose sample() runs the device sampler (sample_gpu.cuh) therefore gets the look-ahead launched from there, right
    // behind the sampler kernel; a caller who takes the greedy pick needs no kernel and gets it launched here, before the wait.
    if (sampler_mode_) spec_deferred_ = true;
    else {
      CTB_CUDA(cudaGraphLaunch(graph_full_, stream_));
      spec_pending_ = true;
    }
  }
}

void Engine::drop_lookahead() { spec_pending_ = false; spec_deferred_ = false; spec_pos_ = -1; spec_streak_ = 0; }

void Engine::launch_deferred_spec() {
  if (!spec_deferred_) return;
  spec_deferred_ = false;
  CTB_CUDA(cudaGraphLaunch(graph_full_, stream_));
  spec_pending_ = true;
}

// The greedy pick of the last eval (what top_k = 1 without a repetition penalty selects, llama.cpp:3832-3857 + 4215-4240: one
// candidate survives, the draw is certain) if the engine computed it: id, or -1 when it did not (look-ahead off, context full,
// non-appending eval) or when several logits share the maximum (std::partial_sort's choice among equals is the reference's).
int Engine::greedy_pick() {
  if (spec_pos_ < 0) return -1;
  DeviceGuard dev_guard(device_);
  CTB_CUDA(cudaEventSynchronize(ev_pick_));
  sampler_mode_ = false;
  launch_deferred_spec();
  const int* pick = h_spec_tok_.as<int>();
  return pick[1] == 1 ? pick[0] : -1;
}

void Engine::put_step(int token, int pos, int n_total) {
  CTB_CUDA(step_ring_.put(stream_, 4, [&](int* st) { st[0] = token; st[1] = pos; st[2] = 0; st[3] = n_total; }));
}

void Engine::decode_one(int token, int pos, int n_total, bool with_logits) {
  put_step(token, pos, n_total);
  CTB_CUDA(cudaGraphLaunch(with_logits ? graph_full_ : graph_nolog_, stream_));
  single_steps_++;
}

int Engine::paths(int* out, int cap) {
  const int v[6] = {fused_ ? 1 : 0, fused_ && ring_attn_ ? 1 : 0, step_slots_, ensure_prefill() ? 1 : 0, (int)prefill_launches_, (int)single_steps_};
  const int n = (int)(sizeof(v) / sizeof(v[0]));
  if (cap < n) return -n;
  std::copy(v, v + n, out);
  return n;
}

void Engine::host_views() {
  eager_ = true;
  if (host_fresh_) return;
  DeviceGuard dev_guard(device_);
  CTB_CUDA(cudaMemcpyAsync(h_logits_.get(), kept_logits_, (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaMemcpyAsync(h_embd_.get(), kept_embd_, (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
  host_fresh_ = true;
}

std::vector<float> Engine::logits_copy() {
  std::vector<float> v((size_t)hp_.n_vocab);
  if (host_fresh_) { memcpy(v.data(), h_logits_.get(), v.size() * 4); return v; }
  DeviceGuard dev_guard(device_);
  CTB_CUDA(cudaMemcpyAsync(v.data(), kept_logits_, v.size() * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
  return v;
}

// Upload the rows' argument block, launch k_sample_topk over them (each on its slot's kept logits) and copy their results back
// (with every slot's greedy pick when `picks`), all on the engine stream; the caller synchronises.
void Engine::sample_enqueue(const SampleRow* rows, int R, bool picks) {
  const int S = hp_.n_seq;
  if (R < 0 || R > S) throw std::runtime_error("device sampler: " + std::to_string(R) + " rows for " + std::to_string(S) + " slots");
  const size_t picks_b = (size_t)S * 8, outs_b = (size_t)S * sizeof(SampleGpuOut);
  const size_t bytes = picks_b + outs_b + sg_block_ints(S, S * SG_MAX_LAST) * 4;
  uint8_t* d_buf = (uint8_t*)d_sample_.grow(bytes);
  uint8_t* h_buf = (uint8_t*)h_sample_.grow(bytes);
  SampleGpuOut* d_out = (SampleGpuOut*)(d_buf + picks_b);
  int* h_blk = (int*)(h_buf + picks_b + outs_b);
  int* d_blk = (int*)(d_buf + picks_b + outs_b);
  int n_tok = 0;
  for (int r = 0; r < R; r++) {
    if (!sg_accepts(rows[r].n_last, rows[r].k) || rows[r].slot < 0 || rows[r].slot >= S) throw std::runtime_error("device sampler: a row it does not take");
    n_tok += sg_window(rows[r].n_last);
  }
  for (int r = 0; r < R; r++) sg_put(h_blk, R, r, rows[r].slot, rows[r].last, rows[r].n_last, rows[r].penalty, rows[r].k, hp_.n_vocab);
  if (R > 0) {
    CTB_CUDA(cudaMemcpyAsync(d_blk, h_blk, sg_block_ints(R, n_tok) * 4, cudaMemcpyHostToDevice, stream_));
    sg_launch(sg_rows(d_blk, R, kept_logits_, (size_t)hp_.n_vocab, d_out), R, hp_.n_vocab, stream_);
    CTB_CUDA(cudaGetLastError());
  }
  // one copy back: the picks (first in the buffer) and then the R results
  if (picks) CTB_CUDA(cudaMemcpyAsync(d_buf, kept_pick_, picks_b, cudaMemcpyDeviceToDevice, stream_));
  const size_t from = picks ? 0 : picks_b, to = picks_b + (size_t)R * sizeof(SampleGpuOut);
  if (to > from) CTB_CUDA(cudaMemcpyAsync(h_buf + from, d_buf + from, to - from, cudaMemcpyDeviceToHost, stream_));
}

int Engine::topk_candidates(const int* last, int n_last, float penalty, int k, int* ids, float* logits) {
  if (!sg_accepts(n_last, k)) return -1;
  DeviceGuard dev_guard(device_);
  sampler_mode_ = true;
  const SampleRow row{0, last, n_last, penalty, k};
  sample_enqueue(&row, 1, false);
  CTB_CUDA(cudaEventRecord(ev_sample_, stream_));
  launch_deferred_spec();                          // the look-ahead step runs while the host finishes the draw
  CTB_CUDA(cudaEventSynchronize(ev_sample_));
  return sg_take(*(const SampleGpuOut*)(h_sample_.as<uint8_t>() + (size_t)hp_.n_seq * 8), ids, logits);
}

void Engine::finish_eval(int next_pos, bool hit) {
  // the look-ahead step (after_eval) overwrites d_logits_ / d_embd_: keep this eval's results where a late request finds them
  CTB_CUDA(cudaMemcpyAsync(kept_logits_, d_logits_, (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToDevice, stream_));
  CTB_CUDA(cudaMemcpyAsync(kept_embd_, d_embd_, (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToDevice, stream_));
  if (eager_) {
    CTB_CUDA(cudaMemcpyAsync(h_logits_.get(), d_logits_, (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToHost, stream_));
    CTB_CUDA(cudaMemcpyAsync(h_embd_.get(), d_embd_, (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToHost, stream_));
  }
  host_fresh_ = eager_;
  CTB_CUDA(cudaEventRecord(ev1_, stream_));
  after_eval(next_pos);
  CTB_CUDA(cudaEventSynchronize(ev1_));
  float ms = 0;
  cudaEventElapsedTime(&ms, ev0_, ev1_);
  stats.last_eval_ms = ms;
  stats.spec_hits += hit ? 1 : 0;
}

// ---- rows of every token (RowSink)
Engine::SinkGuard Engine::rows_begin(const RowSink* rows, int n) {
  sink_ = nullptr; rows_pending_ = 0; rows_done_ = 0; rows_n_ = n;
  if (!rows) return SinkGuard{this};
  if (tp_.world > 1) throw std::runtime_error("the tensor-sharded mode keeps no per-token rows");
  d_rows_.grow((size_t)PB_T * hp_.n_vocab * 4);
  if (rows->targets) {
    if (n > score_cap_) {
      const int cap = std::max(n, 1024);
      d_score_.grow((size_t)cap * 16);
      h_score_.grow((size_t)cap * 16);
      score_cap_ = cap;
    }
    d_lp_ = d_score_.as<double>(); d_tgt_ = (int*)(d_score_.as<uint8_t>() + (size_t)score_cap_ * 8); d_gr_ = d_tgt_ + score_cap_;
    memcpy(h_score_.as<uint8_t>() + (size_t)score_cap_ * 8, rows->targets, (size_t)n * 4);
    CTB_CUDA(cudaMemcpyAsync(d_tgt_, h_score_.as<uint8_t>() + (size_t)score_cap_ * 8, (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
  }
  sink_ = rows;
  return SinkGuard{this};
}

void Engine::rows_take(const float* src, int m) {
  if (rows_done_ + m > rows_n_) throw std::runtime_error("rows: more rows than tokens");
  const size_t nv = (size_t)hp_.n_vocab;
  if (sink_->host) {
    CTB_CUDA(cudaMemcpyAsync(sink_->host + (size_t)rows_done_ * nv, src, (size_t)m * nv * 4, cudaMemcpyDeviceToHost, stream_));
  } else {
    rl_launch(src, m, hp_.n_vocab, d_tgt_ + rows_done_, d_lp_ + rows_done_, d_gr_ + rows_done_, stream_);
    CTB_CUDA(cudaGetLastError());
  }
  rows_done_ += m;
}

void Engine::rows_push(const float* row) {
  CTB_CUDA(cudaMemcpyAsync(d_rows_.as<float>() + (size_t)rows_pending_ * hp_.n_vocab, row, (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToDevice, stream_));
  if (++rows_pending_ == PB_T) rows_drain();
}

void Engine::rows_drain() {
  if (!sink_ || !rows_pending_) return;
  const int m = rows_pending_;
  rows_pending_ = 0;
  rows_take(d_rows_.as<float>(), m);
}

void Engine::rows_finish() {
  if (!sink_) return;
  rows_drain();
  if (rows_done_ != rows_n_) throw std::runtime_error("rows: " + std::to_string(rows_done_) + " rows for " + std::to_string(rows_n_) + " tokens");
  if (sink_->targets) {
    CTB_CUDA(cudaMemcpyAsync(h_score_.get(), d_lp_, (size_t)rows_n_ * 8, cudaMemcpyDeviceToHost, stream_));
    CTB_CUDA(cudaMemcpyAsync(h_score_.as<uint8_t>() + (size_t)score_cap_ * 12, d_gr_, (size_t)rows_n_ * 4, cudaMemcpyDeviceToHost, stream_));
  }
}

void Engine::rows_end() {
  if (sink_ && sink_->targets) {
    if (sink_->logprob) memcpy(sink_->logprob, h_score_.get(), (size_t)rows_n_ * 8);
    if (sink_->greedy) memcpy(sink_->greedy, h_score_.as<uint8_t>() + (size_t)score_cap_ * 12, (size_t)rows_n_ * 4);
  }
}

void Engine::score_kept(int target, double* logprob, int* greedy) {
  DeviceGuard dev_guard(device_);
  RowSink s;
  s.targets = &target; s.logprob = logprob; s.greedy = greedy;
  const SinkGuard sink = rows_begin(&s, 1);
  rows_take(kept_logits_, 1);
  rows_finish();
  CTB_CUDA(cudaStreamSynchronize(stream_));
  rows_end();
}

void Engine::eval_list(const int* tokens, const int* pos, const int* n_total, int n, const RowSink* rows) {
  if (n <= 0) return;
  DeviceGuard dev_guard(device_);
  const SinkGuard sink = rows_begin(rows, n);
  bool hit = false;
  if (spec_pos_ >= 0) {
    const bool was_pending = spec_pending_;   // (a deferred look-ahead nobody launched is simply dropped)
    spec_deferred_ = false;
    bool guessed = false;
    if (n == 1 && pos[0] == spec_pos_ && n_total[0] == pos[0] + 1) {
      CTB_CUDA(cudaEventSynchronize(ev_pick_));
      guessed = h_spec_tok_.as<int>()[0] == tokens[0];
    }
    spec_streak_ = guessed ? spec_streak_ + 1 : 0;
    hit = guessed && was_pending;
    spec_pending_ = false;
    spec_pos_ = -1;
  }
  CTB_CUDA(cudaEventRecord(ev0_, stream_));
  for (int i = 0; i < n; i++) kv_high_ = std::max(kv_high_, pos[i] + 1);
  if (!hit) {
    int i = 0;
    while (i < n) {
      // a run of consecutive positions goes through the batched kernel, PB_T tokens per launch
      int j = i + 1;
      while (j < n && pos[j] == pos[j - 1] + 1 && pos[j] < hp_.n_ctx) j++;
      if (j - i >= prefill_min_ && pos[i] < hp_.n_ctx && ensure_prefill()) {
        for (int b = i; b < j; b += PB_T) {
          const int m = std::min(PB_T, j - b);
          prefill_batch(tokens + b, pos + b, n_total + b, m, b + m == n, sink_ != nullptr);
        }
      } else {
        for (int k = i; k < j; k++) {
          decode_one(tokens[k], pos[k], n_total[k], k == n - 1 || sink_);   // (the full step's body is the same as the short one's)
          if (sink_) rows_push(d_logits_);
        }
      }
      i = j;
    }
  } else if (sink_) {
    rows_push(d_logits_);   // the look-ahead step (graph_full_) computed this token's row
  }   // else: the step for this token at this position is already in the stream
  rows_finish();
  finish_eval(pos[n - 1] + 1, hit);
  rows_end();
}

bool Engine::ensure_prefill() {
  if ((!prefill_on_ && !hp_.multi) || tp_.world > 1) return false;   // (multi-sequence evals have no other path)
  if (pf_ && pf_->tried) return pf_->ok;
  if (!pf_) pf_.reset(new PrefillState());
  PrefillState& P = *pf_;
  P.tried = true;
  for (int i = 0; i < n_body_; i++)
    if (ops_[i].ph.kind == PH_MATVEC && !ops_[i].stream) return false;   // a non-K-quant layer matrix: single-token path only
  const int n_embd = hp_.n_embd, gqa = hp_.n_embd_gqa();
  const int qkvw = n_embd + 2 * gqa;
  // decode buffer -> (batched buffer, floats between token rows)
  struct Map { const float* lo; size_t n; float* b; int ld; };
  std::vector<Map> maps;
  auto add = [&](const float* dec, size_t n) { maps.push_back({dec, n, (float*)P.dalloc((size_t)PB_T * n * 4), (int)n}); };
  add(xa_, n_embd); add(xb_, n_embd); add(qkv_, qkvw); add(attn_, n_embd); add(attn_o_, n_embd); add(ffn_, hp_.n_ff); add(ffn2_, hp_.n_ff);
  auto bat = [&](const float* p, int& ld) -> float* {
    if (!p) { ld = 0; return nullptr; }
    for (const Map& m : maps)
      if (p >= m.lo && p < m.lo + m.n) { ld = m.ld; return m.b + (p - m.lo); }
    throw std::runtime_error("prefill: pointer outside the step workspace");
  };
  P.d_state = (int*)P.dalloc(PB_STATE_MS * 4);
  P.ring = StateRing(P.d_state, PB_STATE_MS, PF_RING);
  std::vector<PPhase>& prog = P.phases;
  int K_max = 0;
  for (int i = 0; i < n_body_; i++) {
    const StepOp& op = ops_[i];
    PPhase ph{};
    ph.state = P.d_state;
    if (op.ph.kind == PH_EMBED) {
      ph.kind = PP_EMBED;
      ph.em = op.ph.em;
      int ld;
      ph.em.out = bat(op.ph.em.out, ld);
      prog.push_back(ph);
    } else if (op.ph.kind == PH_ATTN) {
      ph.at = op.ph.at;
      int ld, ldo;
      ph.at.q = bat(op.ph.at.q, ld); ph.at.k = bat(op.ph.at.k, ld); ph.at.v = bat(op.ph.at.v, ld);
      ph.at.q_stride = ld; ph.at.kv_stride = ld;
      ph.at.out = bat(op.ph.at.out, ldo);
      ph.at.state = P.d_state;
      ph.kind = PP_KV; prog.push_back(ph);
      ph.kind = PP_ATTN; prog.push_back(ph);
    } else {
      K_max = std::max(K_max, op.ph.mv.K);
      pb_matvec_phases(op.ph.mv, (uint8_t*)P.dalloc(pb_qbuf_bytes(op.ph.mv.K)), P.d_state, bat, prog);
    }
  }
  const StepOp& head = ops_[n_body_];
  int ld;
  P.x_final = bat(head.ph.mv.x, ld);
  P.n_body = (int)prog.size();
  P.q3_body = pstep_q3(prog);
  if (head.stream) {   // a K-quant head: the final norm (written as every token's embeddings) and the output matrix over every token
    maps.push_back({d_logits_, (size_t)hp_.n_vocab, (float*)d_rows_.grow((size_t)PB_T * hp_.n_vocab * 4), hp_.n_vocab});
    pb_matvec_phases(head.ph.mv, (uint8_t*)P.dalloc(pb_qbuf_bytes(head.ph.mv.K)), P.d_state, bat, prog);
    P.embd_rows = (float*)P.dalloc((size_t)PB_T * n_embd * 4);
    prog[prog.size() - 2].mv.norm_out = P.embd_rows;
  }
  P.q3_all = pstep_q3(prog);
  P.d_phases = DevMem((prog.size() + 1) * sizeof(PPhase));
  CTB_CUDA(cudaMemset(P.d_phases.get(), 0, (prog.size() + 1) * sizeof(PPhase)));
  CTB_CUDA(cudaMemcpy(P.d_phases.get(), prog.data(), prog.size() * sizeof(PPhase), cudaMemcpyHostToDevice));
  if (!pstep_shape(pb_work_bytes(K_max, hp_.n_ctx, hp_.head_dim()), P.n_slots, P.smem)) return false;
  CTB_CUDA(pstep_set_smem_limit(P.smem));
  P.ok = true;
  return true;
}

// n <= PB_T tokens at consecutive positions through all layers in one launch; `last`: the list ends here, so the head
// mat-vec (logits + final-norm hidden state of the last token) follows on the single-token kernel.
// rows: every token's logits row goes to the sink (RowSink), from the launch's head phases or, for a head that is not a K-quant,
// from head_from per row.
void Engine::prefill_batch(const int* tokens, const int* pos, const int* n_total, int n, bool last, bool rows) {
  PrefillState& P = *pf_;
  MultiTok toks[PB_T];
  for (int i = 0; i < n; i++) toks[i] = MultiTok{0, tokens[i], pos[i], n_total[i], false};
  const bool whole = rows && P.head();
  launch_batch(toks, n, whole);
  prefill_launches_++;
  if (whole) {
    rows_take(d_rows_.as<float>(), n);
  } else if (rows) {
    for (int r = 0; r < n; r++) {
      head_from(P.x_final + (size_t)r * hp_.n_embd);
      rows_push(d_logits_);
    }
  }
  if (last) head_from(P.x_final + (size_t)(n - 1) * hp_.n_embd);
}

// One k_pstep launch of toks[0, n), n <= PB_T: the body, or with `whole` the whole program, whose head phases write every
// token's logits row to d_rows_ (so the single-token rows still waiting there go to the sink first).  The launch state holds
// the token entries (the last one repeated up to PB_T) and n; the multi-sequence build also reads the slot strides and each
// token's slot, the single-sequence build only the first PB_S ints, which are all a single-sequence launch uploads.
void Engine::launch_batch(const MultiTok* toks, int n, bool whole) {
  PrefillState& P = *pf_;
  if (whole) rows_drain();
  size_t kslot, vslot;
  kv_slot_elems(kslot, vslot);
  CTB_CUDA(P.ring.put(stream_, hp_.multi ? PB_STATE_MS : PB_S, [&](int* st) {
    for (int i = 0; i < PB_T; i++) {
      const MultiTok& t = toks[std::min(i, n - 1)];
      st[i * 4] = t.token; st[i * 4 + 1] = t.pos; st[i * 4 + 2] = 0; st[i * 4 + 3] = t.n_total;
      st[PB_S + i] = t.slot;
    }
    st[PB_T * 4] = n; st[PB_T * 4 + 1] = (int)(unsigned)kslot; st[PB_T * 4 + 2] = (int)(unsigned)vslot; st[PB_T * 4 + 3] = 0;
  }));
  CTB_CUDA(P.launch(whole, step_grid_, stream_, d_sync_, hp_.multi));
}

void Engine::head_from(const float* row) {
  const StepOp& head = ops_[n_body_];
  CTB_CUDA(cudaMemcpyAsync(const_cast<float*>(head.ph.mv.x), row, (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToDevice, stream_));
  // just this one op, the way the un-fused schedule launches it
  enqueue_ops(std::vector<StepOp>(1, head), d_prog_ + n_body_, d_bounds_ + (size_t)n_body_ * (sm_count_ + 1), 1, stream_, false);
}

// ---- multi-sequence mode
std::string Engine::multi_refusal() {
  if (tp_.world > 1) return "the tensor-sharded mode";
  for (int i = 0; i < n_body_; i++)
    if (ops_[i].ph.kind == PH_MATVEC && !ops_[i].stream) return "layer matrices that are not K-quants (Q3_K / Q4_K / Q5_K / Q6_K)";
  DeviceGuard dev_guard(device_);
  if (!multi_ready()) return "a context of " + std::to_string(hp_.n_ctx) + " (the batched kernel's attention scratch does not fit in shared memory)";
  return "";
}

bool Engine::multi_ready() { return hp_.multi && ensure_prefill(); }

void Engine::need_multi() {
  if (!multi_ready()) throw std::runtime_error("this engine has no multi-sequence path");
}

void Engine::multi_eval(const std::vector<MultiTok>& toks, const std::vector<int>& starts, const RowSink* rows) {
  DeviceGuard dev_guard(device_);
  need_multi();
  PrefillState& P = *pf_;
  const SinkGuard sink = rows_begin(rows, (int)toks.size());
  const int n_embd = hp_.n_embd, n_vocab = hp_.n_vocab;
  size_t kslot, vslot;
  kv_slot_elems(kslot, vslot);
  if (kslot > 0xffffffffu || vslot > 0xffffffffu) throw std::runtime_error("multi-sequence: a slot's KV region is too large");
  CTB_CUDA(cudaEventRecord(ev0_, stream_));
  for (size_t l = 0; l + 1 < starts.size(); l++) {
    const int a = starts[l], n = starts[l + 1] - a;
    if (n < 1 || n > PB_T) throw std::runtime_error("multi-sequence: bad launch size");
    launch_batch(&toks[a], n, P.head());
    P.m_launches++;
    if (sink_ && P.head()) rows_take(d_rows_.as<float>(), n);   // every token's row of the launch
    for (int r = 0; r < n; r++) {
      const MultiTok& t = toks[a + r];
      if (!t.last && !(sink_ && !P.head())) continue;   // (its logits, if the launch computed them, are dropped)
      float* lg = kept_logits(t.slot);
      float* em = kept_embd(t.slot);
      const float* lsrc = d_logits_;
      const float* esrc = d_embd_;
      if (P.head()) {
        lsrc = d_rows_.as<float>() + (size_t)r * n_vocab;
        esrc = P.embd_rows + (size_t)r * n_embd;
      } else {
        head_from(P.x_final + (size_t)r * n_embd);   // a head that is not a K-quant: k_matvec, one row at a time
        if (sink_) rows_push(d_logits_);
      }
      if (!t.last) continue;
      CTB_CUDA(cudaMemcpyAsync(lg, lsrc, (size_t)n_vocab * 4, cudaMemcpyDeviceToDevice, stream_));
      CTB_CUDA(cudaMemcpyAsync(em, esrc, (size_t)n_embd * 4, cudaMemcpyDeviceToDevice, stream_));
      k_argmax<<<1, ARGMAX_THREADS, 0, stream_>>>(lg, n_vocab, kept_pick_ + 2 * t.slot);
      CTB_CUDA(cudaGetLastError());
    }
  }
  rows_finish();
  CTB_CUDA(cudaEventRecord(ev1_, stream_));
  CTB_CUDA(cudaEventSynchronize(ev1_));
  rows_end();
  float ms = 0;
  cudaEventElapsedTime(&ms, ev0_, ev1_);
  stats.last_eval_ms = ms;
}

void Engine::multi_fetch(int slot, float* logits, float* embd) {
  DeviceGuard dev_guard(device_);
  need_multi();
  CTB_CUDA(cudaMemcpyAsync(logits, kept_logits(slot), (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaMemcpyAsync(embd, kept_embd(slot), (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
}

const SampleGpuOut* Engine::multi_sample(const SampleRow* rows, int R, int* picks) {
  DeviceGuard dev_guard(device_);
  need_multi();
  sample_enqueue(rows, R, true);
  CTB_CUDA(cudaStreamSynchronize(stream_));
  memcpy(picks, h_sample_.get(), (size_t)hp_.n_seq * 8);
  return (const SampleGpuOut*)(h_sample_.as<uint8_t>() + (size_t)hp_.n_seq * 8);
}

void Engine::multi_reset(int slot) {
  DeviceGuard dev_guard(device_);
  zero_slot(slot);
  CTB_CUDA(cudaStreamSynchronize(stream_));
}

long Engine::multi_launches() const { return pf_ ? pf_->m_launches : 0; }

// ---- sequence states
void Engine::kv_slot_elems(size_t& k, size_t& v) const {
  const int hd = hp_.head_dim();
  k = (size_t)hp_.n_layer * hp_.n_ctx * nkv_ * k_stride(hd);
  v = (size_t)hp_.n_layer * kv_ctx_pad(hp_.n_ctx) * nkv_ * hd;
}

void Engine::zero_slot(int slot) {
  size_t k, v;
  kv_slot_elems(k, v);
  CTB_CUDA(cudaMemsetAsync(kc_ + (size_t)slot * k, 0, k * 2, stream_));
  CTB_CUDA(cudaMemsetAsync(vc_ + (size_t)slot * v, 0, v * 2, stream_));
}

void Engine::copy_results(int src, int dst) {
  CTB_CUDA(cudaMemcpyAsync(kept_logits(dst), kept_logits(src), (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToDevice, stream_));
  CTB_CUDA(cudaMemcpyAsync(kept_embd(dst), kept_embd(src), (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToDevice, stream_));
  CTB_CUDA(cudaMemcpyAsync(kept_pick_ + 2 * dst, kept_pick_ + 2 * src, 8, cudaMemcpyDeviceToDevice, stream_));
}

int Engine::state_k_stride() const { return k_stride(hp_.head_dim()); }

// V rows hold position t at v_perm(t), a permutation within each block of 256 positions: a state keeps whole blocks,
// n_pad = n_past rounded up to 256 entries per channel, in the cache's order.
static int v_pad(int n_past) { return (n_past + 255) & ~255; }

// The entries of positions n_past .. n_pad - 1 of every V row are zero in a state, whatever the slot held there (a longer
// history, or the look-ahead step's row at n_past).
static void zero_v_tail(uint16_t* v, size_t rows, int n_past) {
  const int n_pad = v_pad(n_past);
  for (size_t r = 0; r < rows; r++)
    for (int t = n_past; t < n_pad; t++) v[r * n_pad + v_perm(t)] = 0;
}

size_t Engine::state_bytes(int n_past, bool results) const {
  const int hd = hp_.head_dim();
  return (size_t)hp_.n_layer * nkv_ * ((size_t)n_past * k_stride(hd) + (size_t)v_pad(n_past) * hd) * 2 +
         (results ? ((size_t)hp_.n_vocab + hp_.n_embd) * 4 : 0);
}

// K: one 2-D copy of n_layer * n_kv rows (a head's positions are contiguous); V: one of n_layer * n_kv * hd rows (a channel's
// positions are one run of whole 256-blocks).  The host side is the contiguous pinned staging buffer.
void Engine::state_save(int slot, int n_past, bool results, void* out) {
  DeviceGuard dev_guard(device_);
  const int hd = hp_.head_dim(), ks = k_stride(hd);
  size_t kslot, vslot;
  kv_slot_elems(kslot, vslot);
  const size_t rows = (size_t)hp_.n_layer * nkv_, kb = rows * n_past * ks * 2, vb = rows * hd * v_pad(n_past) * 2;
  uint8_t* h = (uint8_t*)h_stage_.grow(std::max<size_t>(state_bytes(n_past, results), 1));
  if (n_past > 0) {
    CTB_CUDA(cudaMemcpy2DAsync(h, (size_t)n_past * ks * 2, kc_ + slot * kslot, (size_t)hp_.n_ctx * ks * 2, (size_t)n_past * ks * 2, rows,
                               cudaMemcpyDeviceToHost, stream_));
    CTB_CUDA(cudaMemcpy2DAsync(h + kb, (size_t)v_pad(n_past) * 2, vc_ + slot * vslot, (size_t)kv_ctx_pad(hp_.n_ctx) * 2, (size_t)v_pad(n_past) * 2,
                               rows * hd, cudaMemcpyDeviceToHost, stream_));
  }
  if (results) {
    CTB_CUDA(cudaMemcpyAsync(h + kb + vb, kept_logits(slot), (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToHost, stream_));
    CTB_CUDA(cudaMemcpyAsync(h + kb + vb + (size_t)hp_.n_vocab * 4, kept_embd(slot), (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToHost, stream_));
  }
  CTB_CUDA(cudaStreamSynchronize(stream_));
  zero_v_tail((uint16_t*)(h + kb), rows * hd, n_past);
  memcpy(out, h, state_bytes(n_past, results));
}

void Engine::state_load(int slot, int n_past, bool results, const void* in, int last_token) {
  DeviceGuard dev_guard(device_);
  const int hd = hp_.head_dim(), ks = k_stride(hd);
  size_t kslot, vslot;
  kv_slot_elems(kslot, vslot);
  const size_t rows = (size_t)hp_.n_layer * nkv_, kb = rows * n_past * ks * 2, vb = rows * hd * v_pad(n_past) * 2;
  float* lg = kept_logits(slot);
  float* em = kept_embd(slot);
  uint8_t* h = (uint8_t*)h_stage_.grow(std::max<size_t>(state_bytes(n_past, results), 1));
  memcpy(h, in, state_bytes(n_past, results));
  zero_v_tail((uint16_t*)(h + kb), rows * hd, n_past);
  if (!hp_.multi) drop_lookahead();   // a look-ahead step may still be in the stream: it runs before the copies below
  zero_slot(slot);
  if (n_past > 0) {
    CTB_CUDA(cudaMemcpy2DAsync(kc_ + slot * kslot, (size_t)hp_.n_ctx * ks * 2, h, (size_t)n_past * ks * 2, (size_t)n_past * ks * 2, rows,
                               cudaMemcpyHostToDevice, stream_));
    CTB_CUDA(cudaMemcpy2DAsync(vc_ + slot * vslot, (size_t)kv_ctx_pad(hp_.n_ctx) * 2, h + kb, (size_t)v_pad(n_past) * 2, (size_t)v_pad(n_past) * 2,
                               rows * hd, cudaMemcpyHostToDevice, stream_));
  }
  if (results) {
    CTB_CUDA(cudaMemcpyAsync(lg, h + kb + vb, (size_t)hp_.n_vocab * 4, cudaMemcpyHostToDevice, stream_));
    CTB_CUDA(cudaMemcpyAsync(em, h + kb + vb + (size_t)hp_.n_vocab * 4, (size_t)hp_.n_embd * 4, cudaMemcpyHostToDevice, stream_));
    if (hp_.multi) {
      k_argmax<<<1, ARGMAX_THREADS, 0, stream_>>>(lg, hp_.n_vocab, kept_pick_ + 2 * slot);
      CTB_CUDA(cudaGetLastError());
    }
  }
  if (!hp_.multi) {
    kv_high_ = n_past;
    host_fresh_ = false;
    if (results && n_past > 0) {
      // as finish_eval leaves an eval of these tokens: the step state at the last token, its results in d_logits_ / d_embd_
      // too, and the greedy pick of the look-ahead (after_eval), whose step then resumes once the caller decodes greedily
      CTB_CUDA(cudaMemcpyAsync(d_logits_, lg, (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToDevice, stream_));
      CTB_CUDA(cudaMemcpyAsync(d_embd_, em, (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToDevice, stream_));
      put_step(last_token, n_past - 1, n_past);
      after_eval(n_past);
    }
  }
  CTB_CUDA(cudaStreamSynchronize(stream_));
}

void Engine::state_fork(int src, const int* dsts, int n) {
  DeviceGuard dev_guard(device_);
  need_multi();
  size_t kslot, vslot;
  kv_slot_elems(kslot, vslot);
  for (int i = 0; i < n; i++) {
    const int d = dsts[i];
    CTB_CUDA(cudaMemcpyAsync(kc_ + d * kslot, kc_ + src * kslot, kslot * 2, cudaMemcpyDeviceToDevice, stream_));
    CTB_CUDA(cudaMemcpyAsync(vc_ + d * vslot, vc_ + src * vslot, vslot * 2, cudaMemcpyDeviceToDevice, stream_));
    copy_results(src, d);
  }
  CTB_CUDA(cudaStreamSynchronize(stream_));
}

// Beam search re-parenting.  Block (lh, c) handles layer / KV head lh of copy c: the K rows of positions [lo, hi), one contiguous
// run of the head's positions, and for every V channel the whole 256-blocks that cover [lo, hi).  V entries are permuted within
// 256-blocks (v_perm), so a whole block is the least that holds every position needed.  The entries below lo it also copies are
// equal in both slots (they hold the same tokens there), and those at hi and above lie past what dst holds, so afterwards dst
// equals src on [0, hi).  No slot is both a source and a destination, so no block reads what another writes.
__global__ void k_kv_reparent(const KvCopy* copies, uint16_t* kc, uint16_t* vc, size_t kslot, size_t vslot, int n_ctx, int ks, int hd) {
  const KvCopy c = copies[blockIdx.y];
  const size_t lh = blockIdx.x;
  const uint4* ksrc = (const uint4*)(kc + c.src * kslot + (lh * n_ctx + c.lo) * ks);
  uint4* kdst = (uint4*)(kc + c.dst * kslot + (lh * n_ctx + c.lo) * ks);
  const int nk = (c.hi - c.lo) * ks / 8;   // (ks is a multiple of 8 halves)
  for (int i = threadIdx.x; i < nk; i += blockDim.x) kdst[i] = ksrc[i];
  const size_t cp = kv_ctx_pad(n_ctx);
  const int v0 = c.lo & ~255, nv = (((c.hi + 255) & ~255) - v0) / 8;
  const uint16_t* vsrc = vc + c.src * vslot + lh * hd * cp + v0;
  uint16_t* vdst = vc + c.dst * vslot + lh * hd * cp + v0;
  for (int i = threadIdx.x; i < hd * nv; i += blockDim.x) {
    const size_t at = (size_t)(i / nv) * cp + (size_t)(i % nv) * 8;
    *(uint4*)(vdst + at) = *(const uint4*)(vsrc + at);
  }
}

size_t Engine::kv_reparent(const std::vector<KvCopy>& copies) {
  DeviceGuard dev_guard(device_);
  need_multi();
  if (copies.empty()) return 0;
  if ((int)copies.size() > hp_.n_seq) throw std::runtime_error("kv_reparent: more copies than slots");
  std::vector<char> src(hp_.n_seq, 0), dst(hp_.n_seq, 0);
  for (const KvCopy& c : copies) {
    if (c.src < 0 || c.src >= hp_.n_seq || c.dst < 0 || c.dst >= hp_.n_seq || c.lo < 0 || c.hi < c.lo || c.hi > hp_.n_ctx)
      throw std::runtime_error("kv_reparent: a copy out of range");
    src[c.src] = 1;
    if (dst[c.dst]++) throw std::runtime_error("kv_reparent: a slot is written twice");
  }
  for (int s = 0; s < hp_.n_seq; s++)
    if (src[s] && dst[s]) throw std::runtime_error("kv_reparent: slot " + std::to_string(s) + " is both a source and a destination");
  KvCopy* d_copies = (KvCopy*)d_copies_.grow(sizeof(KvCopy) * hp_.n_seq);
  KvCopy* h_copies = (KvCopy*)h_copies_.grow(sizeof(KvCopy) * hp_.n_seq);
  const int hd = hp_.head_dim(), ks = k_stride(hd);
  size_t kslot, vslot, bytes = 0;
  kv_slot_elems(kslot, vslot);
  const size_t lh = (size_t)hp_.n_layer * nkv_;
  for (const KvCopy& c : copies) bytes += lh * ((size_t)(c.hi - c.lo) * ks + (size_t)hd * (((c.hi + 255) & ~255) - (c.lo & ~255))) * 2;
  std::copy(copies.begin(), copies.end(), h_copies);
  CTB_CUDA(cudaMemcpyAsync(d_copies, h_copies, sizeof(KvCopy) * copies.size(), cudaMemcpyHostToDevice, stream_));
  k_kv_reparent<<<dim3((unsigned)lh, (unsigned)copies.size()), 256, 0, stream_>>>(d_copies, kc_, vc_, kslot, vslot, hp_.n_ctx, ks, hd);
  CTB_CUDA(cudaGetLastError());
  for (const KvCopy& c : copies) copy_results(c.src, c.dst);
  CTB_CUDA(cudaStreamSynchronize(stream_));
  return bytes;
}

const float* Engine::multi_rows(int slot0, int n) {
  DeviceGuard dev_guard(device_);
  need_multi();
  if (slot0 < 0 || n < 0 || slot0 + n > hp_.n_seq) throw std::runtime_error("multi_rows: slots out of range");
  const size_t b = (size_t)n * hp_.n_vocab * 4;
  float* h = (float*)h_stage_.grow(std::max<size_t>(b, 1));
  CTB_CUDA(cudaMemcpyAsync(h, kept_logits(slot0), b, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
  return h;
}

double Engine::decode_greedy(int first_token, int n_past, int n_steps, int* out_tokens) {
  if (n_steps <= 0) return 0.0;
  drop_lookahead();
  if (n_steps > tokens_out_cap_) throw std::runtime_error("decode_greedy: too many steps");
  if (n_past + n_steps > hp_.n_ctx) throw std::runtime_error("decode_greedy: would run past the context length");
  kv_high_ = std::max(kv_high_, n_past + n_steps);
  DeviceGuard dev_guard(device_);
  put_step(first_token, n_past, n_past + 1);
  CTB_CUDA(cudaEventRecord(ev0_, stream_));
  for (int s = 0; s < n_steps; s++) CTB_CUDA(cudaGraphLaunch(graph_greedy_, stream_));
  CTB_CUDA(cudaEventRecord(ev1_, stream_));
  CTB_CUDA(cudaMemcpyAsync(h_tokens_out_.get(), d_tokens_out_.get(), (size_t)n_steps * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaMemcpyAsync(h_logits_.get(), d_logits_, (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaMemcpyAsync(h_embd_.get(), d_embd_, (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaMemcpyAsync(kept_logits_, d_logits_, (size_t)hp_.n_vocab * 4, cudaMemcpyDeviceToDevice, stream_));
  CTB_CUDA(cudaMemcpyAsync(kept_embd_, d_embd_, (size_t)hp_.n_embd * 4, cudaMemcpyDeviceToDevice, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
  host_fresh_ = true;
  memcpy(out_tokens, h_tokens_out_.get(), (size_t)n_steps * 4);
  float ms = 0;
  cudaEventElapsedTime(&ms, ev0_, ev1_);
  stats.last_eval_ms = ms;
  return ms;
}

// ----------------------------------------------------------------------------- grammar-constrained sampling (grammar_gpu.cuh)
void Engine::grammar_pieces(const std::vector<int>& off, const std::vector<uint8_t>& bytes) {
  if ((int)off.size() != hp_.n_vocab + 1) throw std::runtime_error("grammar pieces: one offset per token and one more are needed");
  DeviceGuard dev_guard(device_);
  const size_t ob = off.size() * 4;
  uint8_t* d = (uint8_t*)d_pieces_.grow(ob + bytes.size() + 1);
  CTB_CUDA(cudaMemcpy(d, off.data(), ob, cudaMemcpyHostToDevice));
  if (!bytes.empty()) CTB_CUDA(cudaMemcpy(d + ob, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
  pieces_ready_ = true;
}

// The launch buffer, the same layout on the device and in pinned memory: the top-k results SampleGpuOut[R], the allowed bits
// [R][gm_words], stats int[R][2] (uploaded as zeros), the k_sample_topk block of the rows with a cut (sample_gpu.cuh sg_put), then the k_grammar_mask block:
// rows [R][GM_ROW_INTS], every grammar's elements and rule offsets (once per grammar), the stacks' nodes, their tops, the windows.
const SampleGpuOut* Engine::grammar_rows(const GrammarRow* rows, int R, int eos, int* stats, unsigned* bits) {
  if (!pieces_ready_) throw std::runtime_error("grammar mask: the vocabulary's pieces are not on the device");
  if (R <= 0 || R > hp_.n_seq) throw std::runtime_error("grammar mask: " + std::to_string(R) + " rows for " + std::to_string(hp_.n_seq) + " slots");
  // the engine's device before the first grow: the buffers below are allocated on the current device, and the engine may run
  // on another one than the caller's (CT_DEVICE, one replica per GPU)
  DeviceGuard dev_guard(device_);
  const int V = hp_.n_vocab;
  std::vector<int> rec((size_t)R * GM_ROW_INTS), elems, roff, nodes, heads, last;
  std::vector<std::pair<const Grammar*, std::pair<int, int>>> seen;   // grammar -> (its first element, its rule offsets' start)
  std::vector<int> cut;                                // rows with a top-k cut
  for (int r = 0; r < R; r++) {
    const GrammarRow& w = rows[r];
    if (w.slot < 0 || w.slot >= hp_.n_seq) throw std::runtime_error("grammar mask: slot out of range");
    // a grammar's elements and rule offsets go into the block once, however many rows use it
    int base = -1, rbase = -1;
    for (const auto& g : seen)
      if (g.first == w.g) { base = g.second.first; rbase = g.second.second; }
    if (base < 0) {
      base = (int)elems.size() / 2;
      rbase = (int)roff.size();
      for (const GElem& x : w.g->elems) { elems.push_back((int)x.type); elems.push_back((int)x.value); }
      for (int o : w.g->off) roff.push_back(base + o);
      seen.push_back({w.g, {base, rbase}});
    }
    int* q = rec.data() + (size_t)r * GM_ROW_INTS;
    q[0] = w.slot;
    q[1] = rbase;
    q[2] = (int)heads.size();
    q[3] = (int)w.s->stacks.size();
    for (const GStack& st : w.s->stacks) {
      int parent = -1;
      for (int e : st) {
        nodes.push_back(base + e);
        nodes.push_back(parent);
        parent = (int)nodes.size() / 2 - 1;
      }
      heads.push_back(parent);
    }
    q[4] = (int)w.s->partial.value;
    q[5] = w.s->partial.n_remain;
    q[6] = w.s->eos_ok() ? 1 : 0;
    const int nl = sg_window(w.n_last);
    q[7] = (int)last.size();
    q[8] = nl;
    last.insert(last.end(), w.last, w.last + nl);
    memcpy(q + 9, &w.penalty, 4);
    if (w.k > 0) {
      if (!sg_accepts(0, w.k)) throw std::runtime_error("grammar mask: a top-k cut the device sampler does not take");
      cut.push_back(r);
    }
  }
  const int C = (int)cut.size();
  const size_t bits_b = (size_t)R * gm_words(V) * 4;
  const size_t outs_b = (size_t)R * sizeof(SampleGpuOut) + bits_b, stats_b = (size_t)R * 8, sg_b = sg_block_ints(C, 0) * 4;
  const size_t gm_ints = rec.size() + elems.size() + roff.size() + nodes.size() + heads.size() + last.size();
  const size_t bytes = outs_b + stats_b + sg_b + gm_ints * 4;
  const size_t res_b = (size_t)R * sizeof(SampleGpuOut);
  uint8_t* d_buf = (uint8_t*)d_gm_.grow(bytes);
  uint8_t* h_buf = (uint8_t*)h_gm_.grow(bytes);
  memset(h_buf + outs_b, 0, stats_b);
  int* h_sg = (int*)(h_buf + outs_b + stats_b);
  for (int c = 0; c < C; c++) sg_put(h_sg, C, c, cut[c], nullptr, 0, 1.0f, rows[cut[c]].k, V);
  int* h = (int*)(h_buf + outs_b + stats_b + sg_b);
  size_t at = 0;
  auto put = [&](const std::vector<int>& v) { const size_t a = at; std::copy(v.begin(), v.end(), h + at); at += v.size(); return a; };
  const size_t o_rec = put(rec), o_el = put(elems), o_roff = put(roff), o_nodes = put(nodes), o_heads = put(heads), o_last = put(last);
  float* scratch = (float*)d_gm_rows_.grow((size_t)R * V * 4);
  sampler_mode_ = true;
  CTB_CUDA(cudaMemcpyAsync(d_buf + outs_b, h_buf + outs_b, bytes - outs_b, cudaMemcpyHostToDevice, stream_));
  const int* d = (const int*)(d_buf + outs_b + stats_b + sg_b);
  const int* pieces = d_pieces_.as<int>();
  GmArgs a{kept_logits_, d + o_rec, (const uint32_t*)(d + o_el), d + o_roff, d + o_nodes, d + o_heads, d + o_last, pieces,
           (const uint8_t*)(pieces + V + 1), scratch, (int*)(d_buf + outs_b), (unsigned*)(d_buf + res_b), V, eos};
  k_grammar_mask<<<dim3((V + GM_THREADS - 1) / GM_THREADS, R), GM_THREADS, 0, stream_>>>(a);
  CTB_CUDA(cudaGetLastError());
  if (C > 0) {
    sg_launch(sg_rows((const int*)(d_buf + outs_b + stats_b), C, scratch, (size_t)V, (SampleGpuOut*)d_buf), C, V, stream_);
    CTB_CUDA(cudaGetLastError());
  }
  CTB_CUDA(cudaMemcpyAsync(h_buf, d_buf, outs_b + stats_b, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaEventRecord(ev_sample_, stream_));
  launch_deferred_spec();                          // the look-ahead step runs while the host finishes the draw
  CTB_CUDA(cudaEventSynchronize(ev_sample_));
  memcpy(stats, h_buf + outs_b, stats_b);
  if (bits) memcpy(bits, h_buf + res_b, bits_b);
  // results in row order: row cut[c]'s cut is at [c]; hand them out at [row]
  std::vector<SampleGpuOut> tmp(cut.size());
  for (int c = 0; c < C; c++) tmp[c] = ((const SampleGpuOut*)h_buf)[c];
  SampleGpuOut* outs = (SampleGpuOut*)h_buf;
  for (int c = 0; c < C; c++) outs[cut[c]] = tmp[c];
  return outs;
}

std::vector<std::vector<float>> Engine::grammar_scratch(const std::vector<int>& rows) {
  std::vector<std::vector<float>> out(rows.size(), std::vector<float>((size_t)hp_.n_vocab));
  DeviceGuard dev_guard(device_);
  for (size_t i = 0; i < rows.size(); i++)
    CTB_CUDA(cudaMemcpyAsync(out[i].data(), d_gm_rows_.as<float>() + (size_t)rows[i] * hp_.n_vocab, out[i].size() * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
  return out;
}

std::vector<float> Engine::slot_logits(int slot) {
  std::vector<float> v((size_t)hp_.n_vocab);
  DeviceGuard dev_guard(device_);
  CTB_CUDA(cudaMemcpyAsync(v.data(), kept_logits(slot), v.size() * 4, cudaMemcpyDeviceToHost, stream_));
  CTB_CUDA(cudaStreamSynchronize(stream_));
  return v;
}

}  // namespace ctb
