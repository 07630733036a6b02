// Eval engine: static device arena + fixed op schedule for the two graph shapes of the path
// (llm_build_llama / llm_build_falcon, reference models/ggml/llama.cpp:2162-2798) driven like
// llama_eval_internal (llama.cpp:2835-2981): last token's logits and post-final-norm hidden state end
// up in host memory owned by the LLM object.
//
// Design: weights repacked once into the stream layout / coalesced planes (device_types.cuh); KV cache fp16;
// a static op list per token whose K-quant mat-vecs, attention, embedding row and greedy pick run as the phases of
// ONE persistent kernel (stream.cuh), replayed as a CUDA graph with {token, n_past} as device scalars; no per-eval
// graph build, no allocator, no thread pool.
#pragma once
#include <cmath>
#include <memory>
#include <string>
#include <vector>

#include "cuda_owned.cuh"
#include "device_types.cuh"
#include "gguf.hpp"

namespace ctb {

// Tensor-sharded mode (SURVEY §8e, BASELINE configs[4]): one process per GPU; rank r of `world` owns the query heads
// [head0, head1) (with their KV heads), the n_ff range [ff0, ff1) — always whole 256-element blocks — and a replica of the
// embedding table, the norms and the output head.  Column-parallel wq / wk / wv / w1 / w3, row-parallel wo / w2, two
// all-reduces of n_embd floats per layer (NCCL over NVLink, captured in the step's CUDA graph).
struct TPShard {
  int rank = 0, world = 1;
  int head0 = 0, head1 = 0, kv0 = 0, kv1 = 0, ff0 = 0, ff1 = 0;
  void* comm = nullptr;   // ncclComm_t
};
// the shard of rank r (same arithmetic as ctransformers_b200/tp_plan.py; throws when the shape does not tile into 256-blocks)
TPShard tp_shard(int n_embd, int n_head, int n_head_kv, int n_ff, int rank, int world);

struct HParams {
  bool falcon = false;
  int n_vocab = 0, n_ctx_train = 0, n_embd = 0, n_ff = 0, n_head = 0, n_head_kv = 0, n_layer = 0, n_rot = 0;
  float eps = 1e-5f, rope_base = 10000.f, rope_scale = 1.f;
  int n_ctx = 512;
  int n_seq = 1;   // sequence slots (KV regions) of the cache; slot 0 has the single-sequence layout
  bool multi = false;   // a multi-sequence handle's engine (ctb_multi_create), whatever its n_seq: evals go through multi_eval
  int head_dim() const { return n_embd / n_head; }
  int n_embd_gqa() const { return head_dim() * n_head_kv; }
};

struct LayerW {
  DevMat wq, wk, wv, wqkv, wo, w1, w2, w3;
  const float* attn_norm = nullptr; const float* attn_norm_b = nullptr;
  const float* attn_norm2 = nullptr; const float* attn_norm2_b = nullptr;
  const float* ffn_norm = nullptr;
};

struct Phase;    // stream.cuh: one phase of the persistent step kernel
struct StepOp;   // engine.cu: one op of the per-token schedule
struct ProfMark; // engine.cu: an event recorded behind a kernel of profile_step, and the kernel's class
struct MVParams;
struct Uploader;
struct PrefillState;

// One token of a multi-sequence eval (multi_pack in llm_abi.cu): its slot, id, position, the row length n_total of its eval
// chunk, and whether its slot's eval ends with it (then its logits are kept).
struct MultiTok { int slot, token, pos, n_total; bool last; };
constexpr int MULTI_LAUNCH_TOKENS = 32;   // tokens of one batched launch (prefill.cuh PB_T)

// One row of the device sampler (sample_gpu.cuh: k_sample_topk): whose logits (a multi-sequence slot; 0 on a single-sequence
// engine), the repetition window, penalty and k.
struct SampleRow { int slot; const int* last; int n_last; float penalty; int k; };

// One row of the grammar mask (grammar_gpu.cuh: k_grammar_mask): whose logits, the grammar and its state (grammar.hpp), the
// repetition window and penalty, and the top-k cut to run on the masked row afterwards (0: none).
struct Grammar;
struct GrammarState;
struct GrammarRow { int slot; const Grammar* g; const GrammarState* s; const int* last; int n_last; float penalty; int k; };

// Where an eval's per-token logits rows go (the reference's logits_all, llama.cpp:2949-2960): every evaluated token's row, in
// call order, either copied to host[i * n_vocab] or reduced on the device by k_row_logprob (score_gpu.cuh) against
// targets[i] into logprob[i] / greedy[i].  Exactly one of host / targets is set.
struct RowSink {
  float* host = nullptr;
  const int* targets = nullptr;
  double* logprob = nullptr;
  int* greedy = nullptr;
};

struct KvCopy { int src, dst, lo, hi; };   // one slot-to-slot KV copy of Engine::kv_reparent

struct EvalStats { double last_eval_ms = 0; long launches = 0; size_t weight_bytes_per_token = 0; long spec_hits = 0; double load_ms = 0; size_t load_bytes = 0; };

class Engine {
 public:
  Engine(const GGUFFile& g, const HParams& hp, int device, const TPShard& tp = TPShard());
  ~Engine();
  Engine(const Engine&) = delete;
  Engine& operator=(const Engine&) = delete;

  // Evaluate a token list with explicit per-token position and n_total (= n_past + N of the reference eval call the token
  // belongs to, llm.h:40-54): consecutive positions go through the batched prefill kernel, PB_T tokens per launch.
  // rows: also keep every token's logits row (RowSink); logits() / embeddings() / the greedy look-ahead come out the same.
  void eval_list(const int* tokens, const int* pos, const int* n_total, int n, const RowSink* rows = nullptr);
  // k_row_logprob on the last eval's kept logits (what logits() holds) against one target
  void score_kept(int target, double* logprob, int* greedy);
  // n_steps greedy decode steps entirely on the device stream (token feedback through k_argmax);
  // out_tokens[n_steps] receives the picked ids.  Returns device-timed milliseconds for the steps.
  double decode_greedy(int first_token, int n_past, int n_steps, int* out_tokens);
  // One eager (un-graphed) decode step at n_past with a CUDA event after every kernel; accumulates the
  // per-class device time.  kinds: 0 mat-vec, 1 attention, 2 rope+kv store, 3 other.  Returns kernel count.
  double time_matvec_only(int reps, long* launches, unsigned mask = 0);
  int profile_step(int token, int n_past, double ms_by_kind[4], int count_by_kind[4]);
  long trace_step(int token, int n_past, unsigned long long* out, long cap_words);
  // Multi-sequence mode (hp.multi): every slot has its own KV region.  multi_refusal: why the model cannot run it, "" when
  // it can.  multi_eval: tokens [starts[i], starts[i+1]) of toks share batched launch i (a slot's tokens within one launch at
  // consecutive positions); afterwards each slot whose eval ended holds its logits, embeddings and greedy pick on the device.
  std::string multi_refusal();
  // rows: the row of every listed token, in the order of toks
  void multi_eval(const std::vector<MultiTok>& toks, const std::vector<int>& starts, const RowSink* rows = nullptr);
  void multi_fetch(int slot, float* logits, float* embd);   // host copies of the slot's last results
  // The device sampler for many slots at once, on the engine stream: one upload of the rows' argument block (pinned), one
  // k_sample_topk launch over them (none when R = 0), one copy back of their results together with every slot's greedy pick
  // (picks[2 * slot] = {arg-max (lowest id), logits equal to the maximum}), one synchronise.  Returns the R results (row r's
  // at [r]), valid until the next call.
  const struct SampleGpuOut* multi_sample(const SampleRow* rows, int R, int* picks);
  void multi_reset(int slot);                               // zero the slot's KV region: a reused slot is a fresh one
  long multi_launches() const;
  // Sequence states (include/ctransformers_b200.h ctb_state_header): the slot's K / V at positions [0, n_past) as
  // K [layer][kv_head][pos][k_stride] then V [layer][kv_channel][pos], fp16, then with `results` its kept logits and embeddings.
  // Every copy is stream-ordered on the engine stream, behind whatever is already in it (a look-ahead step writes position
  // n_past, which a state does not hold).
  size_t state_bytes(int n_past, bool results) const;
  int state_k_stride() const;   // halves of a K row
  void state_save(int slot, int n_past, bool results, void* out);
  // Also zeroes the slot's positions from n_past on, so the slot equals a fresh one that evaluated those tokens.  A
  // single-sequence engine drops its look-ahead and starts over from this state as after an eval ending with last_token.
  void state_load(int slot, int n_past, bool results, const void* in, int last_token);
  void state_fork(int src, const int* dsts, int n);   // multi-sequence: slot src's whole KV region and last results into each dst
  // Beam search re-parenting (multi-sequence): copy i gives slot dst the K rows and V entries of slot src at positions [lo, hi),
  // for every layer and KV head, all copies in one k_kv_reparent launch; then each dst takes src's last results and greedy pick
  // (as state_fork).  No slot may be both a source and a destination.  Returns the K / V bytes the launch moved.
  size_t kv_reparent(const std::vector<KvCopy>& copies);
  // the logits rows of slots [slot0, slot0 + n) in one device-to-host copy, into pinned memory valid until the next call
  const float* multi_rows(int slot0, int n);
  // Which implementations the evals run (include/ctransformers_b200.h ctb_llm_paths): entries written, or -needed.
  int paths(int* out, int cap);
  int step_cluster() const { return step_pair_ ? 2 : 1; }   // CTAs per cluster of the step kernel's launch

  // Host views of the last token's logits / hidden state (the reference hands out ctx->logits.data(), mutable by the caller,
  // llama.cc:47-51).  Until a caller asks for one, nothing is copied per eval (lazy); from the first request on every eval
  // refreshes them, because the caller may keep the pointer.
  float* logits() { host_views(); return h_logits_.as<float>(); }
  float* embeddings() { host_views(); return h_embd_.as<float>(); }
  bool lazy_logits() const { return !eager_; }
  std::vector<float> logits_copy();   // this eval's logits without switching the engine to eager host views
  // Device half of the sampler (sample_gpu.cuh): candidates >= the k-th largest penalised logit.  Returns their count, or -1
  // when the device path does not apply (window too long, k too large, a NaN among the logits, more than SG_MAX_OUT candidates).
  int topk_candidates(const int* last, int n_last, float penalty, int k, int* ids, float* logits);
  // The last eval's greedy pick when the engine has it and it is unambiguous (a unique maximum), else -1.
  int greedy_pick();
  // Grammar-constrained sampling (engine.cu, grammar_gpu.cuh).  grammar_pieces: the vocabulary's pieces, uploaded once (off[n_vocab + 1] into
  // bytes, each piece cut at its first NUL).  grammar_rows: one upload of the rows' argument block (pinned), one k_grammar_mask
  // launch writing each row's penalised, masked logits to scratch row r, one k_sample_topk launch over the scratch rows whose k is
  // not 0 (penalty 1, no window), one copy back, one synchronise.  stats[2 r] = the allowed tokens of row r, stats[2 r + 1] = 1
  // when the device reached a bound on it (its scratch row is then not the mask); bits (optional): the allowed tokens of row r
  // as bits, [R][(n_vocab + 31) / 32].  Returns the top-k results (row r's at [r]), valid until the next call.
  bool has_grammar_pieces() const { return pieces_ready_; }
  void grammar_pieces(const std::vector<int>& off, const std::vector<uint8_t>& bytes);
  const struct SampleGpuOut* grammar_rows(const GrammarRow* rows, int R, int eos, int* stats, unsigned* bits = nullptr);
  // scratch rows of the last grammar_rows call, one copy each and one synchronise for all of them
  std::vector<std::vector<float>> grammar_scratch(const std::vector<int>& rows);
  std::vector<float> slot_logits(int slot);    // a copy of the slot's kept logits
  const HParams& hparams() const { return hp_; }
  EvalStats stats;
  void set_stream(cudaStream_t s);   // run on a caller-owned stream (bench: torch's current stream)
  cudaStream_t stream() const { return stream_; }

 private:
  Engine(const HParams& hp, int device, const TPShard& tp);   // (the public constructor delegates here first: see engine.cu)
  HParams hp_;
  TPShard tp_;
  int nh_ = 0, nkv_ = 0, nff_ = 0;   // this rank's query heads, KV heads and n_ff slice (the whole model when world == 1)
  void tp_all_reduce(float* buf, int n, cudaStream_t st);
  // fused exchange (stream.cuh: XchgParams): this rank's region  uint2 ll[2][world][n_embd]  and every peer's, IPC-mapped
  bool tp_peer_ = false;
  uint8_t* xc_region_ = nullptr;
  uint2* xc_ll_[8] = {nullptr};
  void tp_setup_peer();
  int device_ = 0;
  Stream stream_;
  // arena
  DevMem arena_;
  size_t arena_size_ = 0, arena_used_ = 0;
  void* alloc(size_t bytes, size_t align = 256);

  // weights
  DevMat output_;
  const uint8_t* tok_embd_ = nullptr; int tok_type_ = 0; size_t tok_row_bytes_ = 0;
  const float* out_norm_ = nullptr; const float* out_norm_b_ = nullptr;
  std::vector<LayerW> layers_;
  uint16_t *silu_tab_ = nullptr, *gelu_tab_ = nullptr, *exp_tab_ = nullptr;
  float2* rope_ = nullptr;
  // KV cache
  uint16_t *kc_ = nullptr, *vc_ = nullptr;
  // workspace
  int* d_state_ = nullptr;     // {token, n_past}
  float *xa_ = nullptr, *xb_ = nullptr, *qkv_ = nullptr, *attn_ = nullptr, *attn_o_ = nullptr, *ffn_ = nullptr, *ffn2_ = nullptr, *d_logits_ = nullptr, *d_embd_ = nullptr;
  // every slot's last results (a single-sequence engine's are slot 0's), where a look-ahead step (after_eval) leaves them alone:
  // logits [n_seq][n_vocab], embeddings [n_seq][n_embd], and the multi-sequence slots' greedy picks [n_seq][2] (the single
  // sequence's is the look-ahead's, d_state_ + 4)
  float *kept_logits_ = nullptr, *kept_embd_ = nullptr;
  int* kept_pick_ = nullptr;
  float* kept_logits(int slot) const { return kept_logits_ + (size_t)slot * hp_.n_vocab; }
  float* kept_embd(int slot) const { return kept_embd_ + (size_t)slot * hp_.n_embd; }
  // host (pinned) results
  HostMem h_logits_, h_embd_;
  StateRing step_ring_;        // {token, n_past} of the single-token steps
  void put_step(int token, int pos, int n_total);   // the next ring entry {token, pos, 0, n_total} to d_state_, on the stream
  HostMem h_tokens_out_;
  DevMem d_tokens_out_;
  int tokens_out_cap_ = 0;

  Event ev0_, ev1_, ev_pick_;
  // speculative next step (see after_eval)
  bool spec_on_ = true, spec_pending_ = false;
  bool spec_deferred_ = false;   // a look-ahead step is due but waits for the device sampler to be enqueued first
  bool sampler_mode_ = false;    // the caller's last sample() ran the device sampler kernel (not the greedy pick)
  Event ev_sample_;
  void launch_deferred_spec();
  int spec_pos_ = -1, spec_streak_ = 0;
  void drop_lookahead();         // forget the look-ahead and the streak that earned it (a step already enqueued still runs)
  int kv_high_ = 0;              // one past the highest position any eval has written
  HostMem h_spec_tok_;
  HostMem h_dbg_;                // host-mapped watchdog words of the persistent kernels
  void after_eval(int next_pos);
  int sm_count_ = 132;

  void init(const GGUFFile& g);
  // rows [row0, row1) and K range [k0, k1) of the tensor (defaults: all of it); the shape check is against the FULL tensor
  DevMat upload_matrix(const GGUFTensor& t, struct Uploader& up, int want_K, int want_M, int row0 = 0, int row1 = -1, int k0 = 0, int k1 = -1);
  const float* upload_vector(const GGUFFile& g, const std::string& name, bool required, int want_n);
  // the per-token schedule
  std::vector<StepOp> ops_;      // EMBED, layers..., HEAD, PICK
  int n_body_ = 0;               // ops before the HEAD mat-vec
  Phase* d_prog_ = nullptr;      // device copy of ops_' phases (index = op index)
  Phase* d_prog_mv_ = nullptr;   // scratch program of time_matvec_only
  int *d_bounds_ = nullptr, *d_bounds_mv_ = nullptr;   // per-CTA tile ranges of the two programs
  unsigned* d_sync_ = nullptr;   // grid-barrier words of the step kernel
  int step_grid_ = 0, step_slots_ = 0;   // launch shape of the step kernel: CTAs, ring slots,
  size_t step_smem_ = 0;                 // dynamic shared memory
  bool fused_ = true;            // CTB_STEP_FUSE=0: one kernel per op
  bool step_q3_ = false;         // some mat-vec phase holds a Q3_K matrix: the k_step<.., .., true> build
  bool step_pair_ = false;       // k_step runs as clusters of two CTAs (step_pair_choose)
  bool ring_attn_ = false;       // the step kernel's attention phases take cached K / V through the ring (st_attn_ring_ok)
  void build_ops();
  void push_matvec(struct MVParams& p, int kind);
  void upload_prog(Phase* dst, int* dst_bounds, const std::vector<StepOp>& ops);
  long enqueue_ops(const std::vector<StepOp>& ops, const Phase* d_prog, const int* d_bounds, int n, cudaStream_t st, bool fused,
                   std::vector<ProfMark>* marks = nullptr);
  void build_graphs();
  bool eager_ = false;           // host logits / embeddings are refreshed by every eval
  bool host_fresh_ = true;
  void host_views();
  // the device sampler's buffers, allocated on first use outside the arena for n_seq rows, the same layout on the device and
  // in pinned memory: every slot's greedy pick (int[n_seq][2]), the results (SampleGpuOut[n_seq]), the argument block
  DevMem d_sample_;
  HostMem h_sample_;
  void sample_enqueue(const SampleRow* rows, int R, bool picks);
  // grammar mask: the piece table, the launch buffer (results, stats, argument blocks; device and pinned) and the scratch rows
  bool pieces_ready_ = false;
  DevMem d_pieces_, d_gm_, d_gm_rows_;
  HostMem h_gm_;
  // batched prefill (prefill.cuh): one program, built on first use
  std::unique_ptr<PrefillState> pf_;
  bool multi_ready();            // hp_.multi and the batched program is built
  void need_multi();             // throws unless multi_ready()
  bool prefill_on_ = true;       // CTB_NO_PREFILL=1: prompts run through the single-token kernel
  int prefill_min_ = 4;          // shortest run of consecutive tokens worth a batched launch
  long prefill_launches_ = 0;    // k_pstep launches so far
  long single_steps_ = 0;        // tokens of batch_eval that went through the single-token step
  bool ensure_prefill();
  void prefill_batch(const int* tokens, const int* pos, const int* n_total, int n, bool last, bool rows = false);
  void launch_batch(const MultiTok* toks, int n, bool whole);   // one k_pstep launch: the body, or `whole` with the head phases
  // rows of an eval (RowSink), allocated outside the arena when the batched program or a rows eval first needs them: d_rows_
  // holds up to PB_T rows on their way out, written by a launch's head phases or one at a time (rows_push)
  const RowSink* sink_ = nullptr;
  DevMem d_rows_;
  int rows_pending_ = 0, rows_done_ = 0;
  int rows_n_ = 0;
  DevMem d_score_;               // [cap] doubles logprob, [cap] ints target, [cap] ints greedy; device and pinned
  HostMem h_score_;
  int score_cap_ = 0;
  double* d_lp_ = nullptr;
  int *d_tgt_ = nullptr, *d_gr_ = nullptr;
  struct SinkGuard { Engine* e; ~SinkGuard() { e->sink_ = nullptr; } };
  SinkGuard rows_begin(const RowSink* rows, int n);   // the eval's sink, released when the guard goes (also when the eval throws)
  void rows_finish();                        // enqueue the scores' copy to the host (before finish_eval's event)
  void rows_take(const float* src, int m);   // m rows at src (n_vocab apart) leave for the sink
  void rows_push(const float* row);          // one row through d_rows_
  void rows_drain();
  void rows_end();                           // after the stream is synchronised: the scores to the caller
  void decode_one(int token, int pos, int n_total, bool with_logits);
  void head_from(const float* row);   // the output head (un-fused, as the single-token schedule launches it) on one hidden row
  void finish_eval(int next_pos, bool hit);
  enum : int { MVK_QKV = 0, MVK_WO = 1, MVK_UP = 2, MVK_DOWN = 3, MVK_OUT = 4 };   // which projection a mat-vec launch is
  bool pdl_ = true;              // programmatic dependent launch between the kernels of a step (CTB_NO_PDL=1 turns it off)
  // sequence states
  HostMem h_stage_;              // pinned staging of state_save / state_load, grown on demand
  DevMem d_copies_;              // kv_reparent's copy list (n_seq entries), device and pinned
  HostMem h_copies_;
  void kv_slot_elems(size_t& k, size_t& v) const;   // halves of one slot's K and V regions
  void zero_slot(int slot);                         // zero the slot's K and V regions, on the stream
  void copy_results(int src, int dst);              // multi-sequence: dst takes src's last logits, embeddings and greedy pick
  // the step's graphs, declared last so that they go before the buffers they launch on
  GraphExec graph_full_, graph_nolog_, graph_greedy_;
};

size_t engine_arena_bytes(const GGUFFile& g, const HParams& hp);

}  // namespace ctb
