// Non-matmul stages of the eval graph, each reproducing the reference's rounding points:
//   k_embed     ggml_get_rows on a quantized token_embd            ggml.c:11615-11642 + dequantize_row_* (k_quants.c:784-821, 984-1026, 1123-1166; ggml.c:1483-1610)
//   RoPE        rope_pair / rope_head_pair / rope_k_pair (mode 0 / neox), K row and V channel store   ggml.c:12430-12566, llama.cpp:2303-2335
//   attention   the helpers attn_stage / attn_scores / attn_softmax / attn_vp: RoPE + KV store, K·q (fp16 operands, fp32
//               acc) → scale → causal mask → fp16-table softmax (fp64 sum) → P→fp16 → V·P, with the reference's AVX2
//               f16-dot lane order so the result is bit-exact; composed by attn_body (k_attn and the step kernel's
//               global-memory phase), st_attn_task (stream.cuh) and pb_attn_warp_task (prefill.cuh)
//               llama.cpp:2337-2400, ggml.c:11031 (F16 path), 2392-2426, 11390, 11925-11973, 12009-12078
//   k_argmax    greedy pick on device (used by the fused decode loop; ties → lowest id)
#pragma once
#include <cmath>
#include <vector>

#include "device_types.cuh"

namespace ctb {

// ------------------------------------------------------------------------------------------ embed
// token_embd keeps the GGUF array-of-blocks layout (one row is gathered per token; no streaming access).
__device__ __forceinline__ void k4_scale_min(int j, const uint8_t* q, int& sc, int& m) {
  if (j < 4) { sc = q[j] & 63; m = q[j + 4] & 63; }
  else { sc = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4); m = (q[j + 4] >> 4) | ((q[j] >> 6) << 4); }
}

// Q3 = false: the callers in the kernels of models without Q3_K tensors, which then carry none of its code (see k_step)
template <bool Q3 = true>
__device__ __forceinline__ float dequant_elem(int type, const uint8_t* row, int e) {
  if (Q3 && type == GT_Q3_K) {   // dequantize_row_q3_K (k_quants.c:575-623): block = hmask[32], qs[64], scales[12], d; dl = d·(sc - 32), then dl·q
    const uint8_t* blk = row + (size_t)(e >> 8) * 110;
    const int r = e & 255, n = r >> 7, j = (r & 127) >> 5, l = r & 31, is = 8 * n + 2 * j + (l >> 4);
    const int w = is >> 2, b = is & 3;   // scale word w of the unpacked 16 (k_quants.c:594-598), byte b
    const int lo = w & 1 ? blk[100 + b] : blk[96 + b];
    const int sc = ((w < 2 ? lo : lo >> 4) & 0xF) | (((blk[104 + b] >> (2 * w)) & 3) << 4);
    const int q = ((blk[32 + 32 * n + l] >> (2 * j)) & 3) - ((blk[l] >> (4 * n + j)) & 1 ? 0 : 4);
    return __fmul_rn(__fmul_rn(h2f((uint16_t)(blk[108] | (blk[109] << 8))), (float)(sc - 32)), (float)q);
  }
  switch (type) {
    case GT_F32: return ((const float*)row)[e];
    case GT_F16: return h2f(((const uint16_t*)row)[e]);
    case GT_Q4_0: {
      const uint8_t* blk = row + (size_t)(e >> 5) * 18;
      const int r = e & 31;
      const float d = h2f((uint16_t)(blk[0] | (blk[1] << 8)));
      const int byte = blk[2 + (r & 15)];
      const int nib = r < 16 ? (byte & 0xF) : (byte >> 4);
      return __fmul_rn((float)(nib - 8), d);
    }
    case GT_Q5_0: {   // dequantize_row_q5_0 (ggml.c:1559-1582): block = d, qh[4], qs[16]
      const uint8_t* blk = row + (size_t)(e >> 5) * 22;
      const int r = e & 31;
      const float d = h2f((uint16_t)(blk[0] | (blk[1] << 8)));
      const uint32_t qh = (uint32_t)blk[2] | ((uint32_t)blk[3] << 8) | ((uint32_t)blk[4] << 16) | ((uint32_t)blk[5] << 24);
      const int byte = blk[6 + (r & 15)];
      const int nib = r < 16 ? (byte & 0xF) : (byte >> 4);
      return __fmul_rn((float)((nib | (int)(((qh >> r) & 1u) << 4)) - 16), d);
    }
    case GT_Q4_1: case GT_Q5_1: {   // dequantize_row_q4_1 / q5_1 (ggml.c:1538-1557, 1585-1610): x*d + m, unsigned quants
      const bool q5 = type == GT_Q5_1;
      const uint8_t* blk = row + (size_t)(e >> 5) * (q5 ? 24 : 20);
      const int r = e & 31;
      const float d = h2f((uint16_t)(blk[0] | (blk[1] << 8)));
      const float m = h2f((uint16_t)(blk[2] | (blk[3] << 8)));
      const int byte = blk[(q5 ? 8 : 4) + (r & 15)];
      int q = r < 16 ? (byte & 0xF) : (byte >> 4);
      if (q5) q |= ((blk[4 + (r >> 3)] >> (r & 7)) & 1) << 4;
      return __fmaf_rn((float)q, d, m);   // q*d is exact in fp32, so this equals the reference's x*d + m in either form
    }
    case GT_Q8_0: {
      const uint8_t* blk = row + (size_t)(e >> 5) * 34;
      const float d = h2f((uint16_t)(blk[0] | (blk[1] << 8)));
      return __fmul_rn((float)(int8_t)blk[2 + (e & 31)], d);
    }
    case GT_Q4_K: case GT_Q5_K: {
      const bool q5 = type == GT_Q5_K;
      const uint8_t* blk = row + (size_t)(e >> 8) * (q5 ? 176 : 144);
      const int r = e & 255, j = r >> 6, within = r & 63, sub = 2 * j + (within >> 5), l = within & 31;
      const float d = h2f((uint16_t)(blk[0] | (blk[1] << 8)));
      const float dmin = h2f((uint16_t)(blk[2] | (blk[3] << 8)));
      int sc, m;
      k4_scale_min(sub, blk + 4, sc, m);
      const uint8_t* qs = blk + (q5 ? 48 : 16);
      const int byte = qs[32 * j + l];
      int q = (sub & 1) ? (byte >> 4) : (byte & 0xF);
      if (q5 && (blk[16 + l] & (1 << sub))) q += 16;
      return __fsub_rn(__fmul_rn(__fmul_rn(d, (float)sc), (float)q), __fmul_rn(dmin, (float)m));
    }
    case GT_Q6_K: {
      const uint8_t* blk = row + (size_t)(e >> 8) * 210;
      const uint8_t* ql = blk; const uint8_t* qh = blk + 128; const int8_t* sc = (const int8_t*)(blk + 192);
      const float d = h2f((uint16_t)(blk[208] | (blk[209] << 8)));
      const int r = e & 255, n = r >> 7, rr = r & 127, k = rr >> 5, l = rr & 31, is = l >> 4;
      const int byte = ql[64 * n + ((k & 1) ? 32 : 0) + l];
      const int nib = (k >= 2) ? (byte >> 4) : (byte & 0xF);
      const int hb = (qh[32 * n + l] >> (2 * k)) & 3;
      const int q = (int)(int8_t)(nib | (hb << 4)) - 32;
      return __fmul_rn(__fmul_rn(d, (float)sc[8 * n + is + 2 * k]), (float)q);
    }
  }
  return 0.f;
}

struct EmbedParams { const uint8_t* table; size_t row_bytes; const int* tokens; float* out; int type, K, n_vocab; };

// the embedding row of token id `tok` (clamped to the vocabulary) into out[K], by threads tid, tid + nt, ...
template <bool Q3 = true>
__device__ __forceinline__ void embed_row(const EmbedParams& em, int tok, float* out, int tid, int nt) {
  const uint8_t* row = em.table + (size_t)min(max(tok, 0), em.n_vocab - 1) * em.row_bytes;
  for (int e = tid; e < em.K; e += nt) out[e] = dequant_elem<Q3>(em.type, row, e);
}

// grid = N tokens; out[n][K]
static __global__ void k_embed(const EmbedParams em) {
  embed_row(em, em.tokens[blockIdx.x], em.out + (size_t)blockIdx.x * em.K, threadIdx.x, blockDim.x);
}

// ---------------------------------------------------------------------------------------- rope+kv
// KV cache layouts (ours; the reference keeps K [n_ctx][n_embd_gqa] and V transposed [n_embd_gqa][n_ctx], llama.cpp:2323-2335).
// Both are permuted so that the GPU lane that plays lane L of the reference's 4x8-lane f16 dot (ggml_vec_dot_f16,
// ggml.c:2392-2426: lane L accumulates elements 32i+L in order i) finds ITS elements contiguous:
//   K: [n_kv][n_ctx][k_stride]  head-major (a head's rows of positions 0..T-1 are one contiguous run: one bulk copy brings a
//                               stretch of them into shared memory).  The first np = hd & ~31 elements of a row (the dot's SIMD
//                               part) are lane-major: element e < np at (e & 31) * (np/32) + (e >> 5).  The tail np .. hd-1
//                               (added one by one in double) follows in element order.  The row stride k_stride is hd rounded up
//                               to 8 halves, so that every row and every run of rows is 16-byte aligned for bulk copies and
//                               16-byte loads (hd 64 / 128: stride hd, no tail).
//   V: [n_kv][hd][ctx_pad]      (channel-major like the reference) position t at (t & ~255) + (t & 31) * 8 + ((t >> 5) & 7)
__host__ __device__ inline int kv_ctx_pad(int n_ctx) { return (n_ctx + 255) & ~255; }
__host__ __device__ inline int k_stride(int hd) { return (hd + 7) & ~7; }
// (GEN = false: the caller's hd is 64 or 128, where the stride is hd and there is no tail — the same values in fewer operations)
template <bool GEN = true>
__host__ __device__ inline size_t k_row(int kv_head, int pos, int n_ctx, int hd) { return ((size_t)kv_head * n_ctx + pos) * (GEN ? k_stride(hd) : hd); }   // element offset of a K row
__host__ __device__ inline size_t v_chan(int kv_head, int c, int n_ctx, int hd) { return ((size_t)kv_head * hd + c) * kv_ctx_pad(n_ctx); }   // ... of a V channel
template <bool GEN = true>
__host__ __device__ inline int k_perm(int e, int hd) {
  if (!GEN) return (e & 31) * (hd >> 5) + (e >> 5);
  const int np = hd & ~31;
  return e < np ? (e & 31) * (np >> 5) + (e >> 5) : e;
}
__host__ __device__ inline int v_perm(int t) { return (t & ~255) + (t & 31) * 8 + ((t >> 5) & 7); }

// The (cos, sin) table [n_pos][hd/2] every RoPE kernel reads: the reference's theta recurrence with the same libm calls
// (ggml.c:12482-12529), built on the host once.
inline std::vector<float2> rope_table(int n_pos, int hd, int n_rot, float freq_base, float freq_scale) {
  const int half = hd / 2;
  std::vector<float2> tab((size_t)n_pos * half);
  const float theta_scale = powf(freq_base, -2.0f / n_rot);
  for (int p = 0; p < n_pos; p++) {
    float theta = freq_scale * (float)p;
    for (int i = 0; i < half; i++) {
      tab[(size_t)p * half + i] = make_float2(cosf(theta), sinf(theta));
      theta *= theta_scale;
    }
  }
  return tab;
}

// RoPE of one pair.  mode 0 (llama): x0*c*zeta - x1*s*zeta with the run-time zeta == 1.0f — four separately rounded
// products, no fusion (ggml.c:12521-12539).  neox (falcon): the reference binary contracts the source's x0*c - x1*s and
// x0*s + x1*c into vfmsub231ss / vfmadd132ss (ggml.c:12540-12561 as compiled by gcc -O3 -mfma); verified against the
// compiled reference through ggml_rope_custom_inplace.
__device__ __forceinline__ void rope_pair(float x0, float x1, float2 cs, int neox, float& o0, float& o1) {
  if (neox) {
    o0 = __fmaf_rn(x0, cs.x, -__fmul_rn(x1, cs.y));
    o1 = __fmaf_rn(x0, cs.y, __fmul_rn(x1, cs.x));
  } else {
    o0 = __fsub_rn(__fmul_rn(x0, cs.x), __fmul_rn(x1, cs.y));
    o1 = __fadd_rn(__fmul_rn(x0, cs.y), __fmul_rn(x1, cs.x));
  }
}

// RoPE of pair i of one head's fp32 row x: mode 0 rotates elements i0, i1 = 2i, 2i+1, neox i, i + hd/2 (llama.cpp:2303-2309)
__device__ __forceinline__ void rope_head_pair(const float* x, int i, int hd, int neox, float2 cs, int& i0, int& i1, float& o0, float& o1) {
  i0 = neox ? i : 2 * i;
  i1 = neox ? i + hd / 2 : 2 * i + 1;
  rope_pair(__ldcg(x + i0), __ldcg(x + i1), cs, neox, o0, o1);
}

// the same, rounded to f16 and stored at the pair's K-permuted places of a row, and of a second row when one is given
template <bool GEN = true>
__device__ __forceinline__ void rope_k_pair(const float* x, int i, int hd, int neox, float2 cs, uint16_t* row, uint16_t* row2 = nullptr) {
  int i0, i1;
  float o0, o1;
  rope_head_pair(x, i, hd, neox, cs, i0, i1, o0, o1);
  const uint16_t h0 = f2h(o0), h1 = f2h(o1);
  row[k_perm<GEN>(i0, hd)] = h0; row[k_perm<GEN>(i1, hd)] = h1;
  if (row2) { row2[k_perm<GEN>(i0, hd)] = h0; row2[k_perm<GEN>(i1, hd)] = h1; }
}

// ------------------------------------------------------------------------------------------- attn
// The attention arithmetic, bit-exact with the reference's attention block, written once as the helpers below.  The four
// attention paths compose them in three functions, which differ only in where cached K rows / V channels come from and in
// which threads share a task (NT threads with named barrier BAR, or one warp when NT == 32):
//   attn_body          k_attn (un-fused steps, non-K-quant models) and the step kernel's phase reading global memory
//   st_attn_task       the step kernel's phase with K / V carried by its ring (stream.cuh)
//   pb_attn_warp_task  the batched prefill kernel, one warp per task (prefill.cuh)
// The pieces:
//   attn_stage    RoPE on q and k (the reference's cos/sin recurrence), q -> f16; decode: k, v -> f16 and the cache  (llama.cpp:2303-2335)
//   attn_scores   KQ = ggml_vec_dot_f16(hd, K row, f16(q)) — lane L: fma over elements 32i+L (i < hd/32) in order, then the
//                 4x8 reduce, then elements hd & ~31 .. hd-1 added one by one in double (ggml.c:2392-2426); KQ *= kq_scale
//   attn_softmax  causal soft_max: max, fp16 exp table, fp64 sum (exact), * (float)(1/sum), P -> f16   (ggml.c:12047-12069)
//   attn_vp       KQV = ggml_vec_dot_f16(n_total, V^T row, f16(P)): the first n_total & ~31 positions through the 32 lanes, the
//                 rest added one by one in double — n_total = n_past + N of the eval call the token belongs to (that is the row
//                 length the reference's mul_mat sees, llama.cpp:2373-2385), so results match the reference for the same
//                 batch_size chunking.
// head_dim is any even size from 32 to 256 (attn_head_dim_ok; the engine and the op-level entry points refuse others).  A task
// covers ATTN_CH output channels; the last channel group of a head holds hd % ATTN_CH of them when hd is not a multiple.
struct AttnParams {
  const float* q;        // [N][q_stride] raw projections (NOT yet rotated)
  const float* k;        // [N][kv_stride]
  const float* v;        // [N][kv_stride]
  uint16_t* kc;          // layer K cache
  uint16_t* vc;          // layer V cache
  float* out;            // [N][n_head*hd]
  const uint16_t* exp_tab;
  const float2* rope;    // [n_ctx][hd/2]
  const int* state;      // device: {token, position, step, n_total}
  float kq_scale;
  int n_head, n_kv, hd, n_ctx, q_stride, kv_stride, neox;
};

constexpr int ATTN_THREADS = 512;
constexpr int ATTN_CH = 32;   // output channels per CTA
__host__ __device__ inline int attn_groups(int hd) { return (hd + ATTN_CH - 1) / ATTN_CH; }   // channel groups (tasks) of a head

// Scratch of one task, carved from base:
//   sc  [cp] f32 scores, then exp values         p16 [cp] f16 probabilities, V-permuted order
//   q16 [k_stride] f16 rotated query, K-permuted order
//   cur (decode): k16 [k_stride] f16 rotated key of this position (K-permuted order), v16 [hd] f16 value of this position
// (q16 and k16 are laid out like a K row, so they stay 16-byte aligned)
struct AttnScratch { float* sc; uint16_t *p16, *q16, *k16, *v16; size_t bytes; };
template <bool GEN = true>
__host__ __device__ inline AttnScratch attn_scratch(uint8_t* base, int n_ctx, int hd, bool cur) {
  const size_t cp = kv_ctx_pad(n_ctx), ks = GEN ? k_stride(hd) : hd, end_q = cp * 6 + ks * 2;
  AttnScratch s;
  s.sc = (float*)base;
  s.p16 = (uint16_t*)(base + cp * 4);
  s.q16 = s.p16 + cp;
  s.k16 = cur ? s.q16 + ks : nullptr;
  s.v16 = cur ? s.k16 + ks : nullptr;
  s.bytes = cur ? end_q + ks * 2 + (size_t)hd * 2 : end_q;
  return s;
}
// shared memory of k_attn and of the step kernel's attention phases (the ATTN_CH floats past the scratch are unused; they
// keep the step kernel's shared-memory split, and with it its ring, where it is)
__host__ __device__ inline size_t attn_smem_bytes(int n_ctx, int hd) { return attn_scratch(nullptr, n_ctx, hd, true).bytes + (size_t)ATTN_CH * 4; }

// GGML_F32x8_REDUCE over a warp that plays 4 accumulators x 8 lanes (lane = 8*j + l) — ggml.c:1964-1982
__device__ __forceinline__ float attn_reduce_f32x8(float v) {
  v = v + __shfl_xor_sync(0xffffffffu, v, 16);
  v = v + __shfl_xor_sync(0xffffffffu, v, 8);
  v = v + __shfl_xor_sync(0xffffffffu, v, 4);
  v = v + __shfl_xor_sync(0xffffffffu, v, 1);
  v = v + __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// barrier of the NT threads of a task: named barrier BAR over the first NT threads of the CTA (BAR 0 with NT == blockDim.x is
// __syncthreads), __syncwarp for a warp of its own
template <int BAR, int NT>
__device__ __forceinline__ void attn_bar() {
  if constexpr (NT == 32) __syncwarp();
  else asm volatile("bar.sync %0, %1;" ::"n"(BAR), "n"(NT) : "memory");
}
template <int NT>
__device__ __forceinline__ int attn_tid() { return NT == 32 ? (int)(threadIdx.x & 31) : (int)threadIdx.x; }

// Where the query token with device state st = {token, position, step, n_total} stands: T = pos + 1 scores; V·P runs over the
// eval chunk's n_total positions, the first n_vec = n_total & ~31 through the lanes (t < lim = min(T, n_vec)), the rest in
// double.  T == 0: the position lies past the context, the task does nothing.
struct AttnPos { int pos, T, n_vec, lim; };
__device__ __forceinline__ AttnPos attn_pos(const AttnParams& p, const int* st) {
  AttnPos a;
  a.pos = st[1];
  if (a.pos >= p.n_ctx) { a.T = 0; a.n_vec = 0; a.lim = 0; return a; }
  a.T = a.pos + 1;
  a.n_vec = max(a.T, min(st[3], p.n_ctx)) & ~31;
  a.lim = min(a.T, a.n_vec);
  return a;
}

// rotation of the first pair this thread stages (attn_stage): loaded by the caller, before the wait for q / k / v if it has one
template <int NT>
__device__ __forceinline__ float2 attn_cs0(const AttnParams& p, int pos) {
  const int i = attn_tid<NT>();
  return i < p.hd / 2 ? p.rope[(size_t)pos * (p.hd / 2) + i] : make_float2(1.f, 0.f);
}

// RoPE + f16 of query token n's q for head h into the scratch; with s.k16 (decode) also its k and v.  Then the first query
// head of the KV group writes this position's K row (task cg == 0) and V (every task its ATTN_CH channels) to the cache;
// the task itself takes them from k16 / v16, so there is no ordering hazard.
template <int NT, bool GEN>
__device__ __forceinline__ void attn_stage(const AttnParams& p, const AttnScratch& s, int n, int h, int cg, int pos, float2 cs0) {
  const int hd = p.hd, tid = attn_tid<NT>(), group = p.n_head / p.n_kv, kvh = h / group;
  const bool kv_writer = (h % group) == 0;
  const float* qv = p.q + (size_t)n * p.q_stride + (size_t)h * hd;
  const float* kv = p.k + (size_t)n * p.kv_stride + (size_t)kvh * hd;
  const float* vv = p.v + (size_t)n * p.kv_stride + (size_t)kvh * hd;
  uint16_t* kd = (kv_writer && cg == 0) ? p.kc + k_row<GEN>(kvh, pos, p.n_ctx, hd) : nullptr;
  for (int i = tid; i < hd / 2; i += NT) {
    const float2 cs = i == tid ? cs0 : p.rope[(size_t)pos * (hd / 2) + i];
    rope_k_pair<GEN>(qv, i, hd, p.neox, cs, s.q16);
    if (s.k16) rope_k_pair<GEN>(kv, i, hd, p.neox, cs, s.k16, kd);
  }
  if (s.k16) {
    for (int c = tid; c < hd; c += NT) {
      const uint16_t hv = f2h(__ldcg(vv + c));
      s.v16[c] = hv;
      if (kv_writer && c / ATTN_CH == cg) p.vc[v_chan(kvh, c, p.n_ctx, hd) + v_perm(pos)] = hv;
    }
  }
}

// this lane's PER = hd/32 f16 elements of a K-permuted row, two to a word (PER 2: one word).  Every load is aligned: a row
// starts 16-byte aligned and the lane's elements start at 2 * PER * lane bytes.
template <int PER>
struct KLane { uint32_t w[(PER + 1) / 2]; };
template <int PER>
__device__ __forceinline__ KLane<PER> attn_klane(const uint16_t* row) {
  const uint16_t* p = row + (threadIdx.x & 31) * PER;
  KLane<PER> k;
  if constexpr (PER == 8) {
    const uint4 v = *(const uint4*)p;
    k.w[0] = v.x; k.w[1] = v.y; k.w[2] = v.z; k.w[3] = v.w;
  } else if constexpr (PER == 4) {
    const uint2 v = *(const uint2*)p;
    k.w[0] = v.x; k.w[1] = v.y;
  } else if constexpr (PER % 2 == 0) {
#pragma unroll
    for (int i = 0; i < PER / 2; i++) k.w[i] = ((const uint32_t*)p)[i];
  } else {
#pragma unroll
    for (int i = 0; i < PER / 2; i++) k.w[i] = (uint32_t)p[2 * i] | ((uint32_t)p[2 * i + 1] << 16);
    k.w[PER / 2] = p[PER - 1];
  }
  return k;
}
template <int PER>
__device__ __forceinline__ uint16_t klane_elem(const KLane<PER>& k, int e) { return (uint16_t)((k.w[e >> 1] >> ((e & 1) * 16)) & 0xffff); }
// ... of the rows t0 .. t0+7 of a run of n rows at `rows` (row stride `stride`, clamped to the last row); row `skip` is left 0
template <int PER>
__device__ __forceinline__ void attn_k8(KLane<PER> (&kk)[8], const uint16_t* rows, int stride, int t0, int n, int skip) {
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int t = min(t0 + i, n - 1);
    kk[i] = t == skip ? KLane<PER>{} : attn_klane<PER>(rows + (size_t)t * stride);
  }
}

// Scores of a run of n K rows at `rows` (row stride k_stride(hd)) into sc[0..n).  The warp takes the groups of 8 rows t0 =
// t_first, t_first + t_step, ...; the 8 loads of a group are issued before the first is used (the loop is latency-bound
// otherwise).  Row cur_t (-1: none) comes from `cur` instead of `rows`.  pre, when given, is the first group as
// attn_k8(.., skip = cur_t) loaded it, early.  TAIL: hd may not be 32 * PER; the row's elements 32 * PER .. hd-1 (<= 30 of
// them, the element-ordered tail of the K layout) are added after the lane reduction one by one in double, in element order
// (ggml.c:2415-2418): lane l forms the fp32 product of element 32 * PER + l and the warp adds them in lane order via shuffles.
template <int PER, bool TAIL>
__device__ __forceinline__ void attn_scores_per(const uint16_t* rows, int hd, int n, int t_first, int t_step, const uint16_t* q16, float kq_scale, float* sc,
                                                int cur_t, const uint16_t* cur, const KLane<PER> (*pre)[8]) {
  constexpr int NP = PER * 32;
  constexpr int R = PER > 4 ? 4 : 8;   // rows loaded ahead: a group of 8 in two halves when a lane's share is wider than 8 bytes (registers)
  const int lane = threadIdx.x & 31;
  const int stride = TAIL ? k_stride(hd) : NP, tail = TAIL ? hd - NP : 0;
  const KLane<PER> qq = attn_klane<PER>(q16);
  float q[PER];
#pragma unroll
  for (int e = 0; e < PER; e++) q[e] = h2f(klane_elem(qq, e));
  const float qt = (TAIL && lane < tail) ? h2f(q16[NP + lane]) : 0.f;
  for (int t0 = t_first; t0 < n; t0 += t_step) {
#pragma unroll
    for (int r0 = 0; r0 < 8; r0 += R) {
      KLane<PER> kk[R];
      uint16_t kt[R];
      if (pre && t0 == t_first) {
#pragma unroll
        for (int i = 0; i < R; i++) kk[i] = (*pre)[r0 + i];
      } else {
#pragma unroll
        for (int i = 0; i < R; i++) {
          const int t = min(t0 + r0 + i, n - 1);
          kk[i] = t == cur_t ? KLane<PER>{} : attn_klane<PER>(rows + (size_t)t * stride);
        }
      }
      if constexpr (TAIL) {
#pragma unroll
        for (int i = 0; i < R; i++) {
          const int t = min(t0 + r0 + i, n - 1);
          kt[i] = lane < tail ? (t == cur_t ? cur : rows + (size_t)t * stride)[NP + lane] : (uint16_t)0;
        }
      }
#pragma unroll
      for (int i = 0; i < R; i++)
        if (min(t0 + r0 + i, n - 1) == cur_t) kk[i] = attn_klane<PER>(cur);
#pragma unroll
      for (int i = 0; i < R; i++) {
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < PER; e++) s = __fmaf_rn(h2f(klane_elem(kk[i], e)), q[e], s);
        s = attn_reduce_f32x8(s);
        if constexpr (TAIL) {
          const float term = __fmul_rn(h2f(kt[i]), qt);
          double sumf = (double)s;
          for (int l = 0; l < tail; l++) sumf += (double)__shfl_sync(0xffffffffu, term, l);
          s = (float)sumf;
        }
        if (lane == 0 && t0 + r0 + i < n) sc[t0 + r0 + i] = __fmul_rn(s, kq_scale);
      }
    }
  }
}
// Head sizes 64 / 128 (attn_fast_hd) have kernels of their own; every other size runs in a separate kernel instantiation
// (k_attn<true>, k_step<.., true>) or one out-of-line call (k_pstep), GEN = true below, which keeps its registers out of
// the hot paths of the 64 / 128 kernels.
// F(PER, TAIL) called with the instantiation of head size hd: GEN = false, hd 64 / 128, no tail; GEN = true, any other size,
// with the tail loop (empty when hd is a multiple of 32)
#define ATTN_PER_DISPATCH(GEN, hd, F)                             \
  do {                                                            \
    if constexpr (!(GEN)) {                                       \
      if ((hd) == 128) F(4, false);                               \
      else F(2, false);                                           \
    } else {                                                      \
      switch ((hd) >> 5) {                                        \
        case 1: F(1, true); break;                                \
        case 2: F(2, true); break;                                \
        case 3: F(3, true); break;                                \
        case 4: F(4, true); break;                                \
        case 5: F(5, true); break;                                \
        case 6: F(6, true); break;                                \
        case 7: F(7, true); break;                                \
        default: F(8, true); break;                               \
      }                                                           \
    }                                                             \
  } while (0)
template <bool GEN>
__device__ __forceinline__ void attn_scores(int hd, const uint16_t* rows, int n, int t_first, int t_step, const uint16_t* q16, float kq_scale, float* sc,
                                            int cur_t = -1, const uint16_t* cur = nullptr) {
#define ATTN_SCORES_F(PER, TAIL) attn_scores_per<PER, TAIL>(rows, hd, n, t_first, t_step, q16, kq_scale, sc, cur_t, cur, nullptr)
  ATTN_PER_DISPATCH(GEN, hd, ATTN_SCORES_F);
#undef ATTN_SCORES_F
}

// soft_max of sc[0..T) (ggml.c:12047-12069) -> p16 in V-permuted order, zero up to the end of the last 256-position chunk.
// The NT threads reduce through red_f / red_d [NT/32] (unused by a single warp).  The fp64 sum of fp16 values in (0, 1] is
// exact whatever the grouping.
template <int NT, int BAR>
__device__ __forceinline__ void attn_softmax(float* sc, uint16_t* p16, int T, const uint16_t* exp_tab, float* red_f, double* red_d) {
  constexpr int NW = NT / 32;
  const int tid = attn_tid<NT>(), warp = tid >> 5, lane = tid & 31;
  float mx = -INFINITY;
  for (int t = tid; t < T; t += NT) mx = fmaxf(mx, sc[t]);
  mx = warp_max(mx);
  if constexpr (NW > 1) {
    if (lane == 0) red_f[warp] = mx;
    attn_bar<BAR, NT>();
    mx = red_f[0];
#pragma unroll
    for (int w = 1; w < NW; w++) mx = fmaxf(mx, red_f[w]);
  }
  double sum = 0.0;
  for (int t = tid; t < T; t += NT) {
    const float val = h2f(__ldg(exp_tab + f2h(__fsub_rn(sc[t], mx))));
    sc[t] = val;
    sum += (double)val;
  }
  sum = warp_sum(sum);
  if constexpr (NW > 1) {
    if (lane == 0) red_d[warp] = sum;
    attn_bar<BAR, NT>();
    sum = 0.0;
#pragma unroll
    for (int w = 0; w < NW; w++) sum += red_d[w];
  }
  const float inv = (float)(1.0 / sum);
  const int t_end = (T + 255) & ~255;
  for (int t = tid; t < t_end; t += NT) p16[v_perm(t)] = t < T ? f2h(__fmul_rn(sc[t], inv)) : (uint16_t)0;
  attn_bar<BAR, NT>();
}

// V·P of one output channel, by one warp: vrow = the channel's V, p16 = P, both V-permuted.  Lane part: positions t < lim,
// lane L takes t = 32i+L in increasing i.  Leftover part (ggml.c:2415-2418): positions n_vec <= t < T are added one by one in
// double after the lane reduction.  They are the row i_left of one 256-position chunk, i.e. element i_left of lanes
// 0..T-n_vec-1 of that chunk's 16-byte loads: every lane forms its float product and the warp adds them in lane order through
// shuffles.  Position cur_t (-1: none) takes vcur instead of its cached value; pre, when given, holds the lane's first two
// 256-position chunks of vrow, loaded early.
__device__ __forceinline__ float attn_vp(const uint16_t* vrow, const uint16_t* p16, const AttnPos& a, int cur_t, uint16_t vcur, const uint4* pre = nullptr) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int ch = 0; ch * 256 < a.lim; ch++) {
    uint4 vv;
    if (pre && ch == 0) vv = pre[0];
    else if (pre && ch == 1) vv = pre[1];
    else vv = *(const uint4*)(vrow + ch * 256 + lane * 8);
    const uint4 pp = *(const uint4*)(p16 + ch * 256 + lane * 8);
    const uint32_t vw[4] = {vv.x, vv.y, vv.z, vv.w}, pw[4] = {pp.x, pp.y, pp.z, pp.w};
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int t = ch * 256 + 32 * i + lane;
      if (t < a.lim) {
        uint16_t vh = (uint16_t)((vw[i >> 1] >> ((i & 1) * 16)) & 0xffff);
        const uint16_t ph = (uint16_t)((pw[i >> 1] >> ((i & 1) * 16)) & 0xffff);
        if (t == cur_t) vh = vcur;
        s = __fmaf_rn(h2f(vh), h2f(ph), s);
      }
    }
  }
  s = attn_reduce_f32x8(s);
  double sumf = (double)s;
  const int n_left = a.T - a.n_vec;                   // <= 31; <= 0 when the eval chunk extends past this token
  if (n_left > 0) {
    const int i = (a.n_vec >> 8) * 256 + lane * 8 + ((a.n_vec & 255) >> 5);
    const uint16_t vh = a.n_vec + lane == cur_t ? vcur : vrow[i];
    const float term = __fmul_rn(h2f(vh), h2f(p16[i]));
    for (int l = 0; l < n_left; l++) sumf += (double)__shfl_sync(0xffffffffu, term, l);
  }
  return (float)sumf;
}

// RoPE + KV-cache store + attention for one query token n, one head h and one group cg of ATTN_CH output channels, by NT
// threads with barrier BAR, K / V read from global memory.  Every task of a head recomputes that head's scores (K rows come
// from L2); the channel groups split the V·P work, which gives n_head * ceil(hd/32) tasks per token instead of n_head.
// PDLWAIT = true: a kernel of its own, q/k/v come from the previous kernel (griddepcontrol.wait after the prefetches).
// PDLWAIT = false: a phase of the persistent step kernel (stream.cuh); the caller has already synchronised with the producers.
template <int NT, int BAR, bool PDLWAIT, int PER, bool TAIL>
__device__ __forceinline__ void attn_body_per(const AttnParams& p, uint8_t* smem, const int h, const int n, const int cg, const AttnPos& a,
                                              float* red_f, double* red_d) {
  constexpr int NW = NT / 32;
  // Everything up to pdl_wait() reads only what earlier steps left behind (device state, RoPE table, cached K/V rows of
  // older positions): it overlaps the tail of the QKV kernel.  q/k/v of this token are read after the wait.
  const int hd = p.hd, kvh = h / (p.n_head / p.n_kv), nch = TAIL ? min(ATTN_CH, hd - cg * ATTN_CH) : ATTN_CH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const AttnScratch s = attn_scratch<TAIL>(smem, p.n_ctx, hd, true);
  const uint16_t* krows = p.kc + k_row<TAIL>(kvh, 0, p.n_ctx, hd);
  constexpr int CPW = (ATTN_CH + NW - 1) / NW;          // V channels per warp (the last round may be partial)
  uint4 vpre[CPW][2];                                   // this warp's V rows, first two 256-position chunks
  constexpr bool KPRE = PER <= 4;                       // (a wider share would hold 8 x 16 bytes of registers across the staging)
  KLane<PER> kpre[8];                                   // this warp's first 8 K rows
#pragma unroll
  for (int j = 0; j < CPW; j++)
#pragma unroll
    for (int ch = 0; ch < 2; ch++)
      vpre[j][ch] = (ch * 256 < a.lim && warp + j * NW < nch) ? *(const uint4*)(p.vc + v_chan(kvh, cg * ATTN_CH + warp + j * NW, p.n_ctx, hd) + ch * 256 + lane * 8) : make_uint4(0, 0, 0, 0);
  if constexpr (KPRE) attn_k8<PER>(kpre, krows, TAIL ? k_stride(hd) : PER * 32, warp * 8, a.T, a.pos);
  const float2 cs0 = attn_cs0<NT>(p, a.pos);
  if (PDLWAIT) pdl_wait();

  attn_stage<NT, TAIL>(p, s, n, h, cg, a.pos, cs0);
  attn_bar<BAR, NT>();
  attn_scores_per<PER, TAIL>(krows, hd, a.T, warp * 8, NW * 8, s.q16, p.kq_scale, s.sc, a.pos, s.k16, KPRE ? &kpre : nullptr);
  attn_bar<BAR, NT>();
  attn_softmax<NT, BAR>(s.sc, s.p16, a.T, p.exp_tab, red_f, red_d);
#pragma unroll
  for (int j = 0; j < CPW; j++) {
    const int cc = warp + j * NW;
    if (cc >= nch) break;
    const int c = cg * ATTN_CH + cc;
    const float o = attn_vp(p.vc + v_chan(kvh, c, p.n_ctx, hd), s.p16, a, a.pos, s.v16[c], vpre[j]);
    if (lane == 0) p.out[(size_t)n * p.n_head * hd + (size_t)h * hd + c] = o;
  }
}
// attn_body's reduction slots: one set per CTA size, shared by both GEN forms (a kernel's static shared memory stays as it was)
template <int NT>
__device__ __forceinline__ void attn_body_red(float*& red_f, double*& red_d) {
  __shared__ float rf[NT / 32];
  __shared__ double rd[NT / 32];
  red_f = rf;
  red_d = rd;
}
template <int NT, int BAR, bool PDLWAIT, bool GEN>
__device__ __forceinline__ void attn_body(const AttnParams& p, uint8_t* smem, const int h, const int n, const int cg, const int* st) {
  float* red_f;
  double* red_d;
  attn_body_red<NT>(red_f, red_d);
  const AttnPos a = attn_pos(p, st);
  if (a.T == 0) return;
#define ATTN_BODY_F(PER, TAIL) attn_body_per<NT, BAR, PDLWAIT, PER, TAIL>(p, smem, h, n, cg, a, red_f, red_d)
  ATTN_PER_DISPATCH(GEN, p.hd, ATTN_BODY_F);
#undef ATTN_BODY_F
}

template <bool GEN>
static __global__ void __launch_bounds__(ATTN_THREADS) k_attn(const AttnParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  pdl_trigger();
  attn_body<ATTN_THREADS, 0, true, GEN>(p, smem, blockIdx.x, blockIdx.y, blockIdx.z, p.state);
}
// the k_attn of head size hd
inline void (*attn_kernel(int hd))(const AttnParams) { return attn_fast_hd(hd) ? k_attn<false> : k_attn<true>; }

// ----------------------------------------------------------------------------------------- argmax
// Greedy pick over logits[0, n) by the first NT threads (named barrier BAR): the reference's top_k = 1, a scan that starts at
// element 0 and moves on strictly greater values only.  That is the largest value, the lowest id among equal ones; NaNs never
// win, and id 0 stays picked when nothing exceeds -inf or when logits[0] is NaN.  Thread 0 ends with the result in best / idx.
// CG: the logits were written earlier in the same kernel (read them from L2).
template <int NT, int BAR, bool CG>
__device__ __forceinline__ void block_argmax(const float* logits, int n, float* bv /* [NT / 32] smem */, int* bi /* [NT / 32] smem */, float& best, int& idx) {
  best = -INFINITY;
  idx = 0x7fffffff;
#pragma unroll(CG ? 4 : 1)   // the step kernel's 320 threads keep 4 loads in flight each; k_argmax's 1024 threads need no more registers for it
  for (int i = threadIdx.x; i < n; i += NT) {
    const float v = CG ? __ldcg(logits + i) : logits[i];
    if (v > best) { best = v; idx = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > best || (ov == best && oi < idx)) { best = ov; idx = oi; }
  }
  if ((threadIdx.x & 31) == 0) { bv[threadIdx.x >> 5] = best; bi[threadIdx.x >> 5] = idx; }
  bar_sync<BAR, NT>();
  if (threadIdx.x == 0) {
    for (int w = 1; w < NT / 32; w++)
      if (bv[w] > best || (bv[w] == best && bi[w] < idx)) { best = bv[w]; idx = bi[w]; }
    const float x0 = CG ? __ldcg(logits) : logits[0];
    if (idx == 0x7fffffff || x0 != x0) { best = x0; idx = 0; }   // nothing above -inf, or a NaN at 0 that no value is greater than
  }
}

// the decode state {token, position, step, n_total} after a greedy pick: the pick is the next token (and goes to
// out_tokens[step]); a single-token eval's attention rows have length position + 1
__device__ __forceinline__ void advance_state(int* state, int* out_tokens, int pick) {
  out_tokens[state[2]] = pick;
  state[0] = pick;
  state[1] += 1;
  state[2] += 1;
  state[3] = state[1] + 1;
}

constexpr int ARGMAX_THREADS = 1024;
// single block; writes the greedy pick of block_argmax to out[0] and the number of logits equal to the picked one to out[1] (0 when
// it is a NaN)
static __global__ void k_argmax(const float* logits, int n, int* out) {
  __shared__ float bv[ARGMAX_THREADS / 32];
  __shared__ int bi[ARGMAX_THREADS / 32];
  __shared__ int ties;
  float best;
  int idx;
  block_argmax<ARGMAX_THREADS, 0, false>(logits, n, bv, bi, best, idx);
  if (threadIdx.x == 0) {
    out[0] = idx;
    bv[0] = best;
    ties = 0;
  }
  __syncthreads();
  const float top = bv[0];
  int mine = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) mine += logits[i] == top ? 1 : 0;
  if (mine) atomicAdd(&ties, mine);
  __syncthreads();
  if (threadIdx.x == 0) out[1] = ties;
}

}  // namespace ctb
