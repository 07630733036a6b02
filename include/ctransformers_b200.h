/*
 * ctransformers_b200.h — C ABI of libctransformers.so (H100 / sm_90a build).
 *
 * Part 1 is the reference's own FFI for the hot path, unchanged: the 17 `ctransformers_llm_*`
 * functions that ctransformers/llm.py:117-208 binds with ctypes and that models/llm.cc:32-138 defines.
 * An unmodified `ctransformers` Python package drives this library through
 * `AutoModelForCausalLM.from_pretrained(path, lib="<this .so>")` (lib.py:12-15 returns unknown strings verbatim).
 *
 * Part 2 is additive (`ctb_*`): timing/introspection hooks and op-level entry points with plain
 * host pointers that mirror the ggml operators on the path, so a maintainer (or a parity test) can call
 * one operator at a time.  No torch / CUDA types appear in any signature.
 */
#ifndef CTRANSFORMERS_B200_H_
#define CTRANSFORMERS_B200_H_

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ part 1: reference FFI ---- */
typedef struct LLM LLM; /* opaque; reference: class LLM, models/llm.h:13 */

/* reference: struct Config, models/llm.h:6-11 — passed BY VALUE (ctypes ConfigStruct, llm.py:73-79) */
typedef struct ctransformers_config {
  int context_length; /* <= 0: 512, the llama_context default (llama.cpp:5281) */
  int gpu_layers;     /* ignored: every layer always runs on the GPU */
  bool mmap;          /* ignored: the file is always mmap'ed for the upload */
  bool mlock;         /* ignored */
} ctransformers_config;

/* models/llm.cc:36-76.  GGUF llama / falcon only; NULL (+ stderr) on failure or when no CUDA device exists. */
LLM* ctransformers_llm_create(const char* model_path, const char* model_type, const ctransformers_config config);
void ctransformers_llm_delete(LLM* llm);                                                   /* llm.cc:78  */
/* caller provides room for strlen(text)+1 ints (llm.py:335-337); returns the count */
int ctransformers_llm_tokenize(LLM* llm, const char* text, const bool add_bos_token, int* output); /* llm.cc:80-85 */
const char* ctransformers_llm_detokenize(LLM* llm, const int token);     /* llm.cc:87-89; valid until the next call */
bool ctransformers_llm_is_eos_token(LLM* llm, const int token);          /* llm.cc:91-93  */
int ctransformers_llm_eos_token_id(LLM* llm);                            /* llm.cc:95     */
int ctransformers_llm_bos_token_id(LLM* llm);                            /* llm.cc:97     */
int ctransformers_llm_vocab_size(LLM* llm);                              /* llm.cc:99     */
int ctransformers_llm_context_length(LLM* llm);                          /* llm.cc:101    */
const char* ctransformers_llm_architecture(LLM* llm);                    /* llm.cc:103-105: "llama" | "falcon" */
/* llm.cc:107-112 → LLM::BatchEval (llm.h:40-54).  `threads` is accepted and ignored. */
bool ctransformers_llm_batch_eval(LLM* llm, const int* tokens, const int n_tokens, const int n_past, const int batch_size,
                                  const int threads);
float* ctransformers_llm_logits_data(LLM* llm);             /* llm.cc:114: host, writable, n_vocab floats (last token) */
int ctransformers_llm_logits_size(LLM* llm);                /* llm.cc:116 */
const float* ctransformers_llm_embeddings_data(LLM* llm);   /* llm.cc:118-120: last token's post-final-norm state */
int ctransformers_llm_embeddings_size(LLM* llm);            /* llm.cc:122-124 */
/* llm.cc:126-132 → llama_llm::Sample (llama.cc:53-84) */
int ctransformers_llm_sample(LLM* llm, const int* last_tokens, const int n_last, const int top_k, const float top_p,
                             const float temperature, const float repetition_penalty, int seed);
void ctransformers_llm_reset(LLM* llm);                     /* llm.cc:134 */

/* ------------------------------------------------------------------ part 2: additive ---------- */
int ctb_abi_version(void);
double ctb_llm_last_eval_ms(LLM* llm);              /* CUDA-event time of the last batch_eval / decode_greedy */
long ctb_llm_launches_per_token(LLM* llm);          /* kernels in one decode step's CUDA graph (a K-quant model: 1, the persistent step kernel) */
/* batch_eval calls answered by the step the engine had already started for the greedy next token (engine.cu: after_eval);
 * CTB_NO_SPEC=1 in the environment turns that look-ahead off. */
long ctb_llm_speculative_hits(LLM* llm);
unsigned long long ctb_llm_weight_bytes_per_token(LLM* llm); /* algorithmic weight bytes one decode step reads */
/* sample() calls answered by the device-side repetition penalty + top-k (csrc/sample_gpu.cuh): used while no caller holds a
 * host view of the logits (logits_data / embeddings_data never called); otherwise, or when equal logits make the top-k cut
 * ambiguous, the host sampler runs on the full logits exactly as the reference does. */
long ctb_llm_device_samples(LLM* llm);
/* wall-clock milliseconds the weight upload took (mmap -> pinned staging -> H2D -> repack, pipelined; engine.cu Uploader) */
double ctb_llm_load_ms(LLM* llm);
/* Tensor-sharded mode (BASELINE configs[4]; the reference's closest facility is layer offload to ONE GPU, llm.h:20 gpu_layers —
 * it has no multi-GPU path).  One process per GPU: rank 0 calls ctb_tp_unique_id (128 bytes, a ncclUniqueId) and hands the
 * bytes to the other ranks by any host channel; every rank then calls ctb_llm_create_tp.  Each rank keeps its query heads
 * (with their KV heads) and its n_ff slice, cut on 256-element block boundaries (ctb_tp_shard reports the ranges:
 * head0, head1, kv0, kv1, ff0, ff1), and the step sums two n_embd-float vectors per layer across the ranks — inside the step
 * kernel over NVLink peer memory (CUDA IPC), or with NCCL all-reduce between launches (CTB_TP_NCCL=1).  llama graph only; every rank must make the same calls in the same order and ends up with the same logits. */
int ctb_tp_unique_id(void* out, int cap);                     /* bytes written (128), or -needed */
LLM* ctb_llm_create_tp(const char* model_path, const char* model_type, const ctransformers_config config, int rank, int world,
                       const void* unique_id);
int ctb_tp_shard(int n_embd, int n_head, int n_head_kv, int n_ff, int rank, int world, int* out6);
void ctb_llm_set_stream(LLM* llm, void* cuda_stream);        /* run on a caller-owned cudaStream_t */
/* n_steps greedy decode steps with the token fed back on the device (no host round trip per token);
 * returns the device-timed milliseconds, < 0 on error.  Logits of the last step land in logits_data. */
double ctb_llm_decode_greedy(LLM* llm, int first_token, int n_past, int n_steps, int* out_tokens);

/* One eager decode step, one kernel per op (un-fused), with a CUDA event after every kernel; ADDS device milliseconds and launch counts per class into
 * ms_by_kind[4] / count_by_kind[4] (0 mat-vec, 1 attention, 2 rope+kv store, 3 other).  Returns kernels timed, < 0 on error. */
int ctb_llm_profile_step(LLM* llm, int token, int n_past, double* ms_by_kind, int* count_by_kind);
/* The mat-vec phases of one decode step alone (same kernel, parameters and order; attention, embedding and pick left
 * out), replayed reps times as a CUDA graph between two CUDA events: returns milliseconds per step, < 0 on error;
 * *launches = mat-vec phases per step.  KV cache and logits are not meaningful afterwards. */
/* One fused decode step whose step-kernel CTAs stamp %globaltimer (ns) per phase: out = n_phases x {phase kind, projection},
 * then n_phases x n_cta x {barrier passed, input staged, first weight item in shared memory, phase done}.  Returns the number
 * of phases, 0 if the model does not run fused, or -(words needed). */
long ctb_llm_trace_step(LLM* llm, int token, int n_past, unsigned long long* out, long cap_words);
double ctb_llm_time_matvec_only(LLM* llm, int reps, long* launches);
/* Same, restricted to the launches whose kind bit is set in kind_mask (bit 0 QKV, 1 attention output, 2 FFN gate+up,
 * 3 FFN down, 4 output head; 0 = all): per-projection timing under in-graph launch conditions. */
double ctb_llm_time_matvec_kinds(LLM* llm, int reps, long* launches, unsigned kind_mask);
/* Which implementations this model's evals run, so a caller can tell what a context length and the CTB_* environment
 * switches selected.  out = {decode steps fused into the step kernel (0: one kernel per op, CTB_STEP_FUSE=0), attention of
 * the step kernel fed by its K / V ring (0: attn_body from global memory, or k_attn when not fused), ring slots of the step
 * kernel (ST_W per slot depth), batched prefill available (tries to set it up), batched prefill launches so far, tokens
 * evaluated by single-token steps so far}.  Returns the entries written (6), or -6 when cap is smaller, < 0 on error. */
long ctb_llm_paths(LLM* llm, int* out, int cap);
/* CTAs per cluster the decode-step kernel is launched with: 2 = pairs that stage each mat-vec input together, 1 = single CTAs
 * (CTB_ST_CLUSTER=0, or the GPU or the model does not allow pairs) */
int ctb_llm_step_cluster(LLM* llm);

/* Host-only pieces of the boundary, callable without a GPU: the GGUF vocabulary with its SPM / BPE tokenizer
 * (llama.cpp:1648-1760, 3080-3427, 6151-6187) and the sampler chain of llama_llm::Sample (llama.cc:53-84). */
typedef struct ctb_vocab ctb_vocab;
ctb_vocab* ctb_vocab_load(const char* gguf_path);
void ctb_vocab_free(ctb_vocab* v);
int ctb_vocab_size(ctb_vocab* v);
int ctb_vocab_tokenize(ctb_vocab* v, const char* text, bool add_bos, int* out, int cap); /* count, or -needed if cap is too small */
int ctb_vocab_piece(ctb_vocab* v, int token, char* buf, int cap);                        /* bytes written (no NUL), or -needed */
int ctb_sample(const float* logits, int n_vocab, const int* last_tokens, int n_last, int top_k, float top_p, float temperature,
               float repetition_penalty, int seed);

/* Op-level mirrors (host pointers in, host pointers out; return 0 on success).  ggml type ids: 0 F32, 1 F16,
 * 2 Q4_0, 3 Q4_1, 6 Q5_0, 7 Q5_1, 8 Q8_0, 11 Q3_K, 12 Q4_K, 13 Q5_K, 14 Q6_K (models/ggml/ggml.h enum ggml_type). */
/* ggml_mul_mat for quantized src0 (ggml.c:11031-11245): dst[n*M+m] = dot(W row m, quantize(x col n)). */
int ctb_mul_mat(int type, const void* w_blocks, const float* x, float* dst, int K, int M, int N);
/* quantize_row_q8_K (k_quants.c:1191-1241) / quantize_row_q8_0 (ggml.c:1232-1268): reference block bytes out. */
int ctb_quantize_row_q8_K(const float* x, void* y, int k);
int ctb_quantize_row_q8_0(const float* x, void* y, int k);
/* quantize_row_q8_1 (ggml.c:1420-1481, the activation of Q4_1 / Q5_1 weights): block_q8_1 bytes {float d, float s, int8 qs[32]}. */
int ctb_quantize_row_q8_1(const float* x, void* y, int k);
/* ggml_rms_norm + ggml_mul (mode 1) or ggml_norm + ggml_mul + ggml_add (mode 2) (ggml.c:10674-10720, 10605-10654). */
int ctb_norm(int mode, const float* x, const float* w, const float* b, float* y, int n, float eps);
/* The same norm (mode 1 or 2) through one of the kernels that normalise a mat-vec's input:
 *   path 0  what ctb_norm runs: the prologue of k_matvec (MV_THREADS threads)
 *   path 1  one mat-vec phase of the persistent step kernel launched as the engine launches it (16 all-zero Q4_K rows); y is
 *           the normalised vector CTA 0 writes, as the engine's result_norm / embeddings; n a positive multiple of 256
 * 0 on success, -1 (with a message on stderr) otherwise. */
int ctb_norm_path(int path, int mode, const float* x, const float* w, const float* b, float* y, int n, float eps);
/* CTAs per cluster of the step-kernel launch ctb_norm_path's path 1 makes at width n (2 = a CTA pair stages the input), -1 on error. */
int ctb_norm_path_cluster(int n);
/* ggml_rope_custom on [n_heads][head_dim] at position pos; mode 0 or 2 (neox) (ggml.c:12430-12566). */
int ctb_rope(float* x, int n_heads, int head_dim, int pos, int mode, float freq_base, float freq_scale);
/* One query token (at position T-1) against T cached positions, all heads, exactly as the reference's attention block:
 * KQ (fp16 operands) -> scale -> softmax (fp16 exp table) -> V·P.  Caches in the reference's own layouts:
 * kcache [T][n_kv*hd] fp16 (rotated K), vcache TRANSPOSED [n_kv*hd][T] fp16 (llama.cpp:2323-2335), q [n_head*hd] already
 * rotated, out [n_head*hd].  n_total = n_past + N of the eval call the token belongs to (>= T): the reference's V·P dot runs
 * over rows of that length and splits them at n_total & ~31 between its SIMD lanes and a scalar tail. */
int ctb_attention(const float* q, const uint16_t* kcache, const uint16_t* vcache, float* out, int n_head, int n_kv, int head_dim,
                  int T, int n_total, float kq_scale);
/* n_tok query tokens at positions pos0 .. pos0+n_tok-1 through one of the engine's four attention implementations, each
 * launched the way the engine launches it, RoPE and the KV-cache store included:
 *   path 0  standalone k_attn (un-fused steps, non-K-quant models), one launch per token
 *   path 1  attention phase of the persistent step kernel with cached K / V carried by its shared-memory ring, one launch per
 *           token; fails when the ring cannot carry this n_ctx (st_attn_ring_ok)
 *   path 2  the same phase reading K / V from global memory (attn_body; contexts past the ring's reach), one launch per token
 *   path 3  the batched prefill kernel's KV + attention phases, all tokens in one launch (n_tok <= 32); fails when its
 *           attention scratch does not fit shared memory at this n_ctx
 * q [n_tok][n_head*hd], k_new / v_new [n_tok][n_kv*hd]: projections NOT yet rotated; RoPE mode 0 or 2 (neox), freq_base,
 * freq_scale 1.  kcache [n_ctx][n_kv*hd] fp16 (rotated K) and vcache TRANSPOSED [n_kv*hd][n_ctx] fp16, the reference's layouts
 * (llama.cpp:2323-2335): they hold positions < pos0 on entry and the new tokens' rows as well on return.  n_total[i] = n_past + N
 * of the eval chunk token i belongs to (position + 1 <= n_total[i] <= n_ctx).  out [n_tok][n_head*hd].  0 on success, -1 (with
 * a message on stderr) when the path cannot take the shape. */
int ctb_attention_path(int path, const float* q, const float* k_new, const float* v_new, uint16_t* kcache, uint16_t* vcache,
                       float* out, int n_head, int n_kv, int head_dim, int n_ctx, int pos0, int n_tok, const int* n_total,
                       int rope_mode, float freq_base, float kq_scale);
/* n_tok activation rows through one mat-vec of the batched prefill kernel (k_pstep: its QUANT + GEMM phase pair), launched the
 * way the engine launches it: the engine's grid, the ring depth pstep_shape gives a model of this n_ctx and head_dim, one
 * quantized-activation buffer and PB_T-row token buffers reused by launches of at most 32 tokens (70 tokens run as 32 + 32 + 6).
 * Equals ggml_mul_mat with n_tok columns (ggml.c:11031-11245) plus the engine's prologue and epilogues:
 *   input  row i of x [n_tok][K]; x2 non-null: x * x2 (ggml_mul, the down projection's silu(gate) * up); norm_mode 1 RMSNorm * w,
 *          2 LayerNorm * w + b (norm_w / norm_b [K], eps; a mode ignores what it does not use), 0 none (required with x2); then
 *          quantize_row_q8_K
 *   rows   nseg (1..3) K-quant matrices (types[s] 11 Q3_K, 12 Q4_K, 13 Q5_K, 14 Q6_K; w_blocks[s]: rows[s] rows of K weights in the
 *          reference's block layout) whose outputs sit side by side: out [n_tok][W], W = rows[0] + .. + rows[nseg-1]
 *   epi[s] 0 STORE v, 1 ADD v + res, 3 ADD2 (v + res) + res2, 2 GELU / 4 SILU: the fp16 table of v (ggml.c:3600-3632);
 *          res / res2 [n_tok][W] in out's layout, read only by the segments that add them
 * *n_slots (if non-null) gets the ring slots used.  0 on success, -1 (with a message on stderr) for what the kernel cannot take: a
 * type other than Q3_K / Q4_K / Q5_K / Q6_K, K not a multiple of 256, more than 3 segments, n_tok < 1, or an n_ctx whose attention
 * scratch leaves no ring (the engine then has no batched prefill). */
int ctb_prefill_mul_mat(int nseg, const int* types, const void* const* w_blocks, const int* rows, int K, int n_tok, const float* x,
                        const float* x2, int norm_mode, const float* norm_w, const float* norm_b, float eps, const int* epi,
                        const float* res, const float* res2, float* out, int n_ctx, int head_dim, int* n_slots);
/* n_tok activation rows through one mat-vec phase of a decode step, routed and launched as the engine does it: K-quant matrices
 * (Q3_K / Q4_K / Q5_K / Q6_K) go to the persistent step kernel (k_step), its launch shape chosen as the engine chooses it
 * (clusters of two CTAs that split the input's staging unless CTB_ST_CLUSTER=0, the input is wider than 80 Q8_K blocks, or a
 * matrix is Q3_K); every other type goes to k_matvec with its own activation format (Q8_0, Q8_1, F16 or F32).  Each token is
 * a launch of its own on the same device buffers.  The first arguments and the result are those of ctb_prefill_mul_mat, with
 * any weight type and K a whole number of the types' blocks; then:
 *   norm_out  optional [n_tok][K]: the phase's input after the prologue (the normalised vector, x * x2, or x), as the output
 *             head writes the embeddings
 *   repeat    1..4: the phase runs that many times back to back (one step-kernel program of that many phases, or that many
 *             k_matvec launches); every run writes the same values
 *   launch    output [2] (may be null): {kernel: 1 k_step, 0 k_matvec; CTAs per cluster: 1 or 2}
 * 0 on success, -1 (with a message on stderr) for what the engine never builds: segments of different activation formats, x2
 * with a norm, ADD / ADD2 without res / res2, K not a whole number of blocks, 0 or more than 3 segments, or a K too wide for
 * the step kernel's shared memory. */
int ctb_decode_mul_mat(int nseg, const int* types, const void* const* w_blocks, const int* rows, int K, int n_tok, const float* x,
                       const float* x2, int norm_mode, const float* norm_w, const float* norm_b, float eps, const int* epi,
                       const float* res, const float* res2, float* out, float* norm_out, int repeat, int* launch);
/* silu(W1 x) * (W3 x) with the fp16 SiLU table (ggml.c:3625-3632) — the fused FFN gate. */
int ctb_ffn_gate(int type, const void* w1_blocks, const void* w3_blocks, const float* x, float* out, int K, int M);
/* ggml_get_rows on a quantized table (ggml.c:11615-11642). */
/* How a K-quant mat-vec phase over nseg matrices (types[], rows[], all K wide) is cut up on a GPU with n_sm SMs — pure host
 * arithmetic, no device needed: first_tile[0..grid] = first 16-row tile of each CTA (byte-balanced), meta = {grid, ring slot
 * bytes, tiles alive per CTA (mailboxes), tiles, consumer warps per CTA, rows per tile, work items of the largest CTA,
 * blocks per work item as Q4_K | Q5_K << 8 | Q6_K << 16 | Q3_K << 24}.  0 on success. */
int ctb_matvec_partition(const int* types, const int* rows, int nseg, int K, int n_sm, int* first_tile, int* meta);
/* the paired step kernel's split of a K-wide input's staging: block0[0..2] = first block of cluster rank 0, 1, end; 1 = pairable */
int ctb_stage_pair_split(int K, int* block0);

int ctb_get_row(int type, const void* table_blocks, int K, int n_rows, int row, float* out);

/* The greedy pick of n logits, the reference's top_k = 1 (std::partial_sort of one element: the first largest value; id 0 when
 * nothing exceeds -inf or logits[0] is NaN), through one of the engine's two implementations:
 *   path 0  k_argmax (the look-ahead pick, the un-fused PICK op, each multi-sequence slot's pick): out = {pick, number of logits
 *           equal to the picked one}
 *   path 1  the PH_PICK phase of the persistent step kernel (ctb_llm_decode_greedy's token feedback): out[0..4] is the decode
 *           state {token, position, step, n_total, pick} in and out, advanced as after a greedy step; out[5] = out_tokens[step]
 * 0 on success, -1 (with a message on stderr) for an unknown path or n < 1. */
int ctb_argmax_path(int path, const float* logits, int n, int* out);
/* The device half of the sampler (k_sample_topk), launched as Engine::topk_candidates launches it: the repetition penalty
 * (llama.cpp:4025-4055) over the ids in last_tokens, then every id whose penalised logit is >= the min(k, n)-th largest.  Returns
 * their count (ids / lg get at most 256 of them, in no particular order), -2 when some penalised logit is NaN, -1 for what the
 * kernel does not take (n_last > 256, k < 1, k > 128, n < 1). */
int ctb_sample_topk(const float* logits, int n, const int* last_tokens, int n_last, float repetition_penalty, int k, int* ids, float* lg);
/* ctransformers_llm_sample's chain for logits that live on the device, on an uploaded copy of logits: the greedy shortcut on a
 * unique k_argmax pick, else the device top-k when its cut is unambiguous, else the host sampler on all logits.  Returns the
 * token (the one ctb_sample draws with the same arguments), -1 on error; *used_device = 1 when the device answered. */
int ctb_sample_device(const float* logits, int n, const int* last_tokens, int n_last, int top_k, float top_p, float temperature,
                      float repetition_penalty, int seed, int* used_device);
/* Both of the above on n_rows rows of n logits each (logits[r * n ..]), row r with the window last_tokens[last_off[r] ..
 * last_off[r + 1]) and its own settings, launched as ctb_multi_sample_many launches them: one k_sample_topk launch over the rows.
 * ctb_sample_topk_rows: count[r] as ctb_sample_topk returns it (-2 NaN, -1 for a window or k the kernel does not take: that row
 *   is not launched), its ids / logits at ids[r * 256 ..] / lg[r * 256 ..].
 * ctb_sample_device_rows: tokens[r] as ctb_sample_device draws it with seed[r], used_device[r] its flag.
 * 0, or -1 (+ stderr) for no rows, n < 1 or window offsets that are not ascending. */
int ctb_sample_topk_rows(const float* logits, int n_rows, int n, const int* last_off, const int* last_tokens, const float* repetition_penalty,
                         const int* k, int* count, int* ids, float* lg);
int ctb_sample_device_rows(const float* logits, int n_rows, int n, const int* last_off, const int* last_tokens, const int* top_k, const float* top_p,
                           const float* temperature, const float* repetition_penalty, const int* seed, int* tokens, int* used_device);

/* Multi-sequence decoding: one handle owns n_slots sequence slots, each of which behaves like a fresh single-sequence LLM with
 * the same config, and every eval's slots share batched launches (one pass over the weights per launch of up to 32 tokens).
 * After every eval a slot's logits, embeddings, greedy pick and sampler draws are bit-identical to what a single-sequence LLM
 * returns for that slot's own call history.  The KV cache holds one region per slot ([slot][layer][kv_head][pos][k_stride]).
 * Runs models whose layer matrices are all K-quants at contexts where the batched kernel fits (not at 4096 and above); create
 * returns NULL (+ stderr) otherwise, without a CUDA device, in a process that holds a tensor-sharded rank, and when the n_slots
 * KV regions do not fit (the message gives the bytes needed). */
typedef struct ctb_multi ctb_multi;
ctb_multi* ctb_multi_create(const char* model_path, const char* model_type, const ctransformers_config config, int n_slots);
void ctb_multi_delete(ctb_multi* m);
int ctb_multi_info(ctb_multi* m, int* out6);   /* {n_slots, n_vocab, n_embd, context length, eos id, bos id}; returns 6 */
/* slot slots[i] evaluates tokens[off[i] .. off[i+1]) at n_past[i], chunked by batch_size as ctransformers_llm_batch_eval
 * chunks; all listed slots (each at most once) share launches.  false (+ stderr) on error. */
bool ctb_multi_eval(ctb_multi* m, int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size);
const float* ctb_multi_logits(ctb_multi* m, int slot);       /* n_vocab floats of the slot's last eval; NULL before one */
const float* ctb_multi_embeddings(ctb_multi* m, int slot);   /* n_embd floats */
/* greedy picks (= sample with top_k 1, no penalty) of n slots from the device arg-max; 0, or -1 (+ stderr) on error */
int ctb_multi_greedy(ctb_multi* m, int n, const int* slots, int* out);
/* = ctransformers_llm_sample on that slot's logits (RNG reseeded per call); -1 (+ stderr, e.g. for a slot out of range or
 * without logits) on error.  ctb_multi_sample_many of one slot. */
int ctb_multi_sample(ctb_multi* m, int slot, const int* last_tokens, int n_last, int top_k, float top_p, float temperature,
                     float repetition_penalty, int seed);
/* out[i] = ctransformers_llm_sample on slot slots[i]'s logits with the window last_tokens[last_off[i] .. last_off[i + 1]),
 * top_k[i], top_p[i], temperature[i], repetition_penalty[i] and seed[i] (the RNG reseeded per slot, in list order; < 0: time).
 * Each draw is the one a single-sequence LLM with that slot's history returns.  The penalty and top-k cut of every slot run in
 * one device launch and one copy back; the host finishes each draw from its candidates, or on the slot's logits where the
 * device cannot answer (a window over 256 tokens, top_k outside 1 .. 128, equal logits at the cut, NaN).  0, or -1 (+ stderr)
 * for a slot out of range, listed twice or without logits, or window offsets that are not ascending: checked before the first
 * draw, so nothing is drawn then. */
int ctb_multi_sample_many(ctb_multi* m, int n, const int* slots, const int* last_off, const int* last_tokens, const int* top_k, const float* top_p,
                          const float* temperature, const float* repetition_penalty, const int* seed, int* out);
long ctb_multi_device_samples(ctb_multi* m);     /* draws of sample / sample_many / greedy answered on the device so far */
int ctb_multi_reset(ctb_multi* m, int slot);    /* the slot starts over; 0, or -1 when out of range */
long ctb_multi_launches(ctb_multi* m);           /* batched launches so far */
double ctb_multi_last_eval_ms(ctb_multi* m);     /* CUDA-event time of the last eval */
/* Host only: the token list ctb_multi_eval makes of these arguments, out[i] = {slot, position, n_total, launch, last of its
 * slot's eval} (5 ints per token).  Returns the token count, or -count when cap is smaller. */
int ctb_multi_pack(int n, const int* slots, const int* off, const int* n_past, int batch_size, int n_ctx, int* out, int cap);

/* Sequence states: what a sequence has evaluated, as one self-describing blob that moves between slots of a handle, between
 * handles of the same file whatever their context lengths and slot counts, and between LLM and ctb_multi.  Little-endian:
 *   ctb_state_header
 *   int32  tokens[n_tokens]                                 n_past = n_tokens
 *   fp16   K[n_layer][n_head_kv][n_past][k_stride]          rotated K rows as the cache holds them (k_stride = head_dim rounded up
 *                                                           to a multiple of 8: the first head_dim & ~31 channels lane-major, the
 *                                                           rest in order, then zeros)
 *   fp16   V[n_layer][n_head_kv * head_dim][n_pad]          V transposed, one row of positions per channel, in whole blocks of
 *                                                           256 (n_pad = n_past rounded up to 256) permuted as the cache holds
 *                                                           them: position t at (t & ~255) + (t & 31) * 8 + ((t >> 5) & 7);
 *                                                           the entries of positions n_past .. n_pad - 1 are zero
 *   float  logits[n_vocab], embeddings[n_embd]              only when has_results: the last eval's
 * The fingerprint hashes (64-bit FNV-1a) the GGUF metadata, the tensor table and the first 4 KiB of every tensor's data, so a
 * state of another file is refused even when the shapes agree.  A restore zeroes the positions from n_past on, so the slot equals
 * a fresh one that evaluated the tokens; it needs n_past <= the context length.  Refusals (bad magic or version, a size that
 * disagrees with the header, another model, n_past above the context) return -1 with the reason on stderr and leave the slot or
 * LLM as it was.  The tensor-sharded mode has no states. */
#define CTB_STATE_MAGIC 0x53425443u /* "CTBS" */
#define CTB_STATE_VERSION 1u
typedef struct ctb_state_header {
  uint32_t magic, version;
  int32_t n_layer, n_head_kv, head_dim, k_stride, n_embd, n_vocab;
  int32_t n_tokens;    /* n_past */
  int32_t has_results; /* 0 or 1 */
  uint64_t fingerprint;
} ctb_state_header;
/* Host only: checks a blob's header and that size is exactly what it describes; 0 and *out filled, or -1 (+ stderr). */
int ctb_state_info(const void* buf, size_t size, ctb_state_header* out);
size_t ctb_llm_state_size(LLM* llm, int n_tokens);                 /* bytes of the state after these tokens; 0 on error */
/* the LLM's state after it has evaluated tokens[0 .. n_tokens) (its n_past); 0, or -1 (+ stderr), e.g. when cap is smaller */
int ctb_llm_save_state(LLM* llm, const int* tokens, int n_tokens, void* buf, size_t cap);
/* After a load, sample and batch_eval behave as after an ordinary eval of the state's tokens, the greedy look-ahead included. */
int ctb_llm_load_state(LLM* llm, const void* buf, size_t size);
size_t ctb_multi_state_size(ctb_multi* m, int n_tokens);
int ctb_multi_save(ctb_multi* m, int slot, const int* tokens, int n_tokens, void* buf, size_t cap);
int ctb_multi_restore(ctb_multi* m, int slot, const void* buf, size_t size);
/* Device to device: each of slots dsts[0 .. n) becomes a byte-identical copy of slot src (its whole KV region, last results and
 * greedy pick), stream-ordered.  src must not be among dsts.  0, or -1 (+ stderr). */
int ctb_multi_fork(ctb_multi* m, int src, int n, const int* dsts);

/* Beam search: the reference's llama_beam_search (llama.cpp:4334-4579) driven as its examples/beam_search does (a beam is at its
 * end when its last token is EOS), each result bit-identical.  Prompt i (tokens [prompt_off[i], prompt_off[i + 1])) is evaluated
 * in one slot, chunked by batch_size as ctransformers_llm_batch_eval chunks it; its search holds n_beams slots, and prompts are
 * admitted as slots free up.  Each step evaluates every live beam of every prompt in one batched eval; the beams are chosen on
 * the host from their logits rows; then one launch moves K / V between slots where beams re-parent.  The response of prompt i
 * (at most n_predict tokens, an EOS included when the winning beam ends in one) goes to out_tokens[out_off[i] .. out_off[i + 1])
 * (room for n_prompts * n_predict ids, out_off for n_prompts + 1), the winner's renormalised p to out_p[i].  The slots used
 * are reset afterwards.  0, or -1 (+ stderr) with every slot usable: n_beams outside 1 .. min(n_slots, n_vocab), an empty
 * prompt, a prompt whose length plus n_predict exceeds the context, a token id out of range, or a continuation whose p
 * underflows to 0 (undefined in the reference). */
int ctb_multi_beam_search(ctb_multi* m, int n_prompts, const int* prompt_off, const int* prompt_tokens, int n_beams, int n_predict, int batch_size,
                          int* out_off, int* out_tokens, float* out_p);
/* the last beam search: steps, host-clock ms of the evals, of the row fetches + selections and of the re-parentings, the K / V
 * bytes the re-parenting launches moved, the tokens evaluated (prompts included), the steps that also evaluated a prompt and
 * the ms of their evals */
int ctb_multi_beam_stats(ctb_multi* m, double* out8);
/* Op level, for tests.  One selection step of the beam search on given rows: n_in beams (p, eob) with their logits rows
 * ([n_in][n_vocab]; an eob beam's row is unused), n_next entries left from the step before (0 at the first step, then the
 * previous step's beam count).  Writes the new beams in the reference's array order: the index of the beam each comes from,
 * the token it adds (-1: an eob beam carried over), its renormalised p and eob flag.  Returns their count, or -1 (+ stderr),
 * e.g. when a continuation's p underflows to 0. */
int ctb_beam_step(int n_beams, int n_in, int n_next, const float* in_p, const unsigned char* in_eob, const float* rows, int n_vocab, int* out_parent,
                  int* out_token, float* out_p, unsigned char* out_eob);
/* Op level, for tests: the re-parenting launch of the beam search.  Slot dst[i] takes slot src[i]'s K / V at positions
 * [lo[i], hi[i]) (whole 256-position blocks of V), its last results and greedy pick; no slot may be both a source and a
 * destination.  Returns the K / V bytes moved, or -1 (+ stderr). */
long ctb_multi_reparent(ctb_multi* m, int n, const int* src, const int* dst, const int* lo, const int* hi);

/* Rows of every token: the logits row of every evaluated token, not only the last one's, each bit-identical to what the
 * reference's llama_eval returns for that token with the context flag logits_all set (llama.cpp:2949-2960), under the same
 * batch_size chunking and n_past clamp as ctransformers_llm_batch_eval.  Otherwise an eval with rows is an ordinary eval:
 * logits_data, embeddings_data (the last token's only, as in the reference), the greedy look-ahead and sample come out the same.
 *
 * ctb_llm_batch_eval_rows: ctransformers_llm_batch_eval that also writes token i's n_vocab logits to rows[i * n_vocab].
 * ctb_llm_batch_eval_scored: the same eval, each row reduced on the device against targets[i] (-1: none) to
 *   logprob[i] = (double)l[t] - m - log(sum_j exp((double)l[j] - m)),  m = the row's largest logit, and
 *   greedy[i]  = 1 when targets[i] is the row's greedy pick (sample with top_k = 1: the lowest id of the largest logit), else 0;
 *   only 12 bytes per token come back to the host.  The order of the sum and the results for rows with NaN or infinities are
 *   those of k_row_logprob (csrc/score_gpu.cuh): NaN in the row gives NaN; +inf entries share the mass; all -inf gives NaN;
 *   no target gives logprob 0, greedy 0.
 * ctb_llm_score_last: that reduction of the last eval's logits (what logits_data holds) against one target.
 * ctb_row_logprob: the same kernel on n_rows host rows (op level).
 * ctb_multi_eval_rows / ctb_multi_eval_scored: ctb_multi_eval with every listed token's row or score, in the order of the
 *   concatenated token lists (tokens[off[0]] first); targets is aligned with it.
 * 0 on success, -1 (+ stderr) on failure.  A target outside -1 .. n_vocab - 1, a token id out of range, or the tensor-sharded
 * mode (which keeps no rows) is refused before anything runs, and the handle stays usable. */
int ctb_llm_batch_eval_rows(LLM* llm, const int* tokens, int n_tokens, int n_past, int batch_size, float* rows);
int ctb_llm_batch_eval_scored(LLM* llm, const int* tokens, int n_tokens, int n_past, int batch_size, const int* targets, double* logprob,
                              int* greedy);
int ctb_llm_score_last(LLM* llm, int target, double* logprob, int* greedy);
int ctb_row_logprob(const float* rows, int n_rows, int n_vocab, const int* targets, double* logprob, int* greedy);
int ctb_multi_eval_rows(ctb_multi* m, int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size, float* rows);
int ctb_multi_eval_scored(ctb_multi* m, int n, const int* slots, const int* off, const int* tokens, const int* n_past, int batch_size,
                          const int* targets, double* logprob, int* greedy);

/* ---- grammar-constrained sampling (csrc/grammar.hpp, csrc/grammar_gpu.cuh): the reference's llama_sample_grammar and
 * llama_grammar_accept_token over grammars in the GBNF text format of its grammar_parser::parse.
 *
 * ctb_grammar_parse: NULL on refusal (a syntax error, no `root`, a rule referenced but never defined, left recursion), with the
 *   message in err (cap bytes, NUL-terminated) and the byte offset where parsing stopped in *err_pos.
 * ctb_grammar_info: {n_rules, n_elements, n_symbols}.  ctb_grammar_rules: rule r is elements[off[r] .. off[r + 1]) of
 *   elems (type, value pairs: llama_grammar_element).  ctb_grammar_symbol: symbol i (in id order): its name (bytes written, or
 *   -needed) and *id.
 * A state (stacks + partial UTF-8 sequence) keeps its grammar alive.  ctb_grammar_start: the state llama_grammar_init gives.
 * ctb_grammar_accept_piece / ctb_llm_grammar_accept / ctb_multi_grammar_accept: llama_grammar_accept_token with the piece given,
 *   or the model's piece of token; 0, or -1 (+ stderr) when the state does not allow the token (the state is left as it was).
 * ctb_grammar_mask_pieces: the host mask over n_vocab pieces (piece t = bytes[off[t] .. off[t + 1])): allowed[t] = 1 where
 *   llama_sample_grammar leaves token t's logit finite.
 * ctb_llm_grammar_mask / ctb_multi_grammar_mask: that mask over the model's vocabulary, computed by k_grammar_mask on the
 *   device (a row the device cannot finish is answered by the host code).
 * ctb_llm_sample_grammar: ctransformers_llm_sample with llama_sample_grammar between the repetition penalty and top-k; the token,
 *   or -1 (+ stderr) when no token is allowed or the handle is tensor-sharded.
 * ctb_multi_sample_grammar_many: ctb_multi_sample_many with state states[i] for draw i (NULL: unconstrained, drawn as
 *   ctb_multi_sample_many draws); every constrained row goes into one k_grammar_mask launch.
 * ctb_llm_grammar_paths / ctb_multi_grammar_paths: out3 = {constrained draws the device answered, rows the host masked because
 *   the device reached a bound, draws whose top-k cut the host made on the masked row (fewer allowed tokens than top_k, or an
 *   ambiguous cut)}. */
typedef struct ctb_grammar ctb_grammar;
typedef struct ctb_grammar_state ctb_grammar_state;
ctb_grammar* ctb_grammar_parse(const char* text, char* err, int cap, long* err_pos);
void ctb_grammar_free(ctb_grammar* g);
int ctb_grammar_info(const ctb_grammar* g, int* out3);
int ctb_grammar_rules(const ctb_grammar* g, int* off, unsigned* elems);
int ctb_grammar_symbol(const ctb_grammar* g, int i, char* name, int cap, unsigned* id);
ctb_grammar_state* ctb_grammar_start(const ctb_grammar* g);
ctb_grammar_state* ctb_grammar_state_copy(const ctb_grammar_state* s);
void ctb_grammar_state_free(ctb_grammar_state* s);
int ctb_grammar_state_eos_ok(const ctb_grammar_state* s);
int ctb_grammar_state_stacks(const ctb_grammar_state* s, int* out, int cap, int* partial2);   /* ints written, or -needed */
int ctb_grammar_accept_piece(ctb_grammar_state* s, const char* piece, int len, int is_eos);
int ctb_llm_grammar_accept(LLM* llm, ctb_grammar_state* s, int token);
int ctb_multi_grammar_accept(ctb_multi* m, ctb_grammar_state* s, int token);
int ctb_grammar_mask_pieces(const ctb_grammar_state* s, int n_vocab, const int* off, const char* bytes, int eos, unsigned char* allowed);
int ctb_llm_grammar_mask(LLM* llm, const ctb_grammar_state* s, unsigned char* allowed);
int ctb_multi_grammar_mask(ctb_multi* m, int slot, const ctb_grammar_state* s, unsigned char* allowed);
int ctb_llm_sample_grammar(LLM* llm, const int* last_tokens, int n_last, int top_k, float top_p, float temperature, float repetition_penalty,
                           int seed, const ctb_grammar_state* s);
int ctb_multi_sample_grammar_many(ctb_multi* m, int n, const int* slots, const int* last_off, const int* last_tokens, const int* top_k,
                                  const float* top_p, const float* temperature, const float* repetition_penalty, const int* seed,
                                  const ctb_grammar_state* const* states, int* out);
int ctb_llm_grammar_paths(LLM* llm, long* out3);
int ctb_multi_grammar_paths(ctb_multi* m, long* out3);

#ifdef __cplusplus
}
#endif
#endif /* CTRANSFORMERS_B200_H_ */
