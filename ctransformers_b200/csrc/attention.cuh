// Non-matmul stages of the eval graph, each reproducing the reference's rounding points:
//   k_embed     ggml_get_rows on a quantized token_embd            ggml.c:11615-11642 + dequantize_row_* (k_quants.c:784-821, 984-1026, 1123-1166; ggml.c:1483-1608)
//   k_rope_kv   RoPE (mode 0 / neox) in place on Q, on K → fp16 KV  ggml.c:12430-12566, llama.cpp:2303-2335
//   k_attn      K·q (fp16 operands, fp32 acc) → scale → causal mask → fp16-table softmax (fp64 sum) → P→fp16 → V·P, with
//               the reference's AVX2 f16-dot lane order so the result is bit-exact
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

__device__ __forceinline__ float dequant_elem(int type, const uint8_t* row, int e) {
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

// grid = N tokens; out[n][K]
static __global__ void k_embed(const uint8_t* table, int type, size_t row_bytes, int K, int n_vocab, const int* tokens, float* out) {
  const int tok = tokens[blockIdx.x];
  const uint8_t* row = table + (size_t)min(max(tok, 0), n_vocab - 1) * row_bytes;
  float* o = out + (size_t)blockIdx.x * K;
  for (int e = threadIdx.x; e < K; e += blockDim.x) o[e] = dequant_elem(type, row, e);
}

// ---------------------------------------------------------------------------------------- rope+kv
// KV cache layouts (ours; the reference keeps K [n_ctx][n_embd_gqa] and V transposed [n_embd_gqa][n_ctx], llama.cpp:2323-2335).
// Both are permuted so that the GPU lane that plays lane L of the reference's 4x8-lane f16 dot (ggml_vec_dot_f16,
// ggml.c:2392-2426: lane L accumulates elements 32i+L in order i) finds ITS elements contiguous:
//   K: [n_kv][n_ctx][hd]        head-major (a head's rows of positions 0..T-1 are one contiguous run: one bulk copy brings a
//                               stretch of them into shared memory); element e of a row is stored at (e & 31) * (hd/32) + (e >> 5)
//   V: [n_kv][hd][ctx_pad]      (channel-major like the reference) position t at (t & ~255) + (t & 31) * 8 + ((t >> 5) & 7)
__host__ __device__ inline int kv_ctx_pad(int n_ctx) { return (n_ctx + 255) & ~255; }
__host__ __device__ inline size_t k_row(int kv_head, int pos, int n_ctx, int hd) { return ((size_t)kv_head * n_ctx + pos) * hd; }   // element offset of a K row
__host__ __device__ inline int k_perm(int e, int hd) { return (e & 31) * (hd >> 5) + (e >> 5); }
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

struct RopeKVParams {
  float* q;             // [N][n_head*hd]   rotated in place
  const float* k;       // [N][n_kv*hd]
  const float* v;       // [N][n_kv*hd]
  uint16_t* kc;         // this layer's K cache (RoPE'd K, llama.cpp:2333)
  uint16_t* vc;         // this layer's V cache
  const float2* rope;   // [n_ctx][hd/2] (cos, sin), built on the host with libm exactly like the reference loop
  const int* state;     // device: {token, position, step, n_total}
  int n_head, n_kv, hd, n_ctx, neox;
  int q_stride, kv_stride;   // row strides (floats) of q and k/v — falcon reads them out of one fused qkv row
};

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

// grid = (N, n_head + n_kv), block = hd/2
static __global__ void k_rope_kv(const RopeKVParams p) {
  const int n = blockIdx.x, hh = blockIdx.y, i = threadIdx.x;
  const int pos = p.state[1] + n;
  if (pos >= p.n_ctx) return;
  const float2 cs = p.rope[(size_t)pos * (p.hd / 2) + i];
  const int i0 = p.neox ? i : 2 * i, i1 = p.neox ? i + p.hd / 2 : 2 * i + 1;
  if (hh < p.n_head) {
    float* qh = p.q + (size_t)n * p.q_stride + (size_t)hh * p.hd;
    float o0, o1;
    rope_pair(qh[i0], qh[i1], cs, p.neox, o0, o1);
    qh[i0] = o0; qh[i1] = o1;
  } else {
    const int kh = hh - p.n_head;
    const float* ksrc = p.k + (size_t)n * p.kv_stride + (size_t)kh * p.hd;
    const float* vsrc = p.v + (size_t)n * p.kv_stride + (size_t)kh * p.hd;
    float o0, o1;
    rope_pair(ksrc[i0], ksrc[i1], cs, p.neox, o0, o1);
    uint16_t* kd = p.kc + k_row(kh, pos, p.n_ctx, p.hd);
    kd[k_perm(i0, p.hd)] = f2h(o0);
    kd[k_perm(i1, p.hd)] = f2h(o1);
    const int cp = kv_ctx_pad(p.n_ctx);
    uint16_t* vd = p.vc + (size_t)kh * p.hd * cp + v_perm(pos);
    vd[(size_t)(2 * i) * cp] = f2h(vsrc[2 * i]);
    vd[(size_t)(2 * i + 1) * cp] = f2h(vsrc[2 * i + 1]);
  }
}

// ------------------------------------------------------------------------------------------- attn
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
constexpr int ATTN_WARPS = ATTN_THREADS / 32;
constexpr int ATTN_CH = 32;   // output channels per CTA

__host__ __device__ inline size_t attn_smem_bytes(int n_ctx, int hd) {
  return (size_t)kv_ctx_pad(n_ctx) * 6 + (size_t)hd * 2 * 3 + (size_t)ATTN_CH * 4;
}

// GGML_F32x8_REDUCE over a warp that plays 4 accumulators x 8 lanes (lane = 8*j + l) — ggml.c:1964-1982
__device__ __forceinline__ float attn_reduce_f32x8(float v) {
  v = v + __shfl_xor_sync(0xffffffffu, v, 16);
  v = v + __shfl_xor_sync(0xffffffffu, v, 8);
  v = v + __shfl_xor_sync(0xffffffffu, v, 4);
  v = v + __shfl_xor_sync(0xffffffffu, v, 1);
  v = v + __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// Fused RoPE + KV-cache store + attention for one query token (blockIdx.y), one head (blockIdx.x) and one group of
// ATTN_CH output channels (blockIdx.z), bit-exact with the reference's attention block:
//   RoPE on q and k (k_rope table = the reference's cos/sin recurrence), K -> f16 cache, V -> f16 cache  (llama.cpp:2303-2335)
//   KQ  = ggml_vec_dot_f16(hd, K row, f16(q))  — lane L: fma over elements 32i+L in order, then the 4x8 reduce
//   KQ *= kq_scale; causal mask; soft_max: max, fp16 exp table, fp64 sum (exact), * (float)(1/sum)   (ggml.c:12047-12069)
//   KQV = ggml_vec_dot_f16(n_total, V^T row, f16(P)): the first n_total & ~31 positions through the 32 lanes, the rest added
//         one by one in double — n_total = n_past + N of the eval call the token belongs to (that is the row length the
//         reference's mul_mat sees, llama.cpp:2373-2385), so results match the reference for the same batch_size chunking.
// Every CTA of a head recomputes that head's scores (K rows come from L2); the channel groups split the V·P work, which
// gives n_head * hd/32 CTAs per token instead of n_head.  The CTA with blockIdx.z == 0 of the first head of each KV group
// writes that group's K row; V channels are written by the CTAs (first head of the group) that own them.  The current
// position is always taken from the freshly computed k/v, never read back from the cache, so there is no ordering hazard.
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// named barrier over the first NT threads of the CTA (BAR 0 with NT == blockDim.x is __syncthreads)
template <int BAR, int NT>
__device__ __forceinline__ void attn_bar() { asm volatile("bar.sync %0, %1;" ::"n"(BAR), "n"(NT) : "memory"); }

// NT threads (barrier BAR) work on one (query token n, head, channel group) task; q/k/v rows of token n are at n * stride.
// PDLWAIT = true: a kernel of its own, q/k/v come from the previous kernel (griddepcontrol.wait after the prefetches).
// PDLWAIT = false: a phase of the persistent step kernel (stream.cuh); the caller has already synchronised with the producers.
template <int NT, int BAR, bool PDLWAIT>
__device__ __forceinline__ void attn_body(const AttnParams& p, uint8_t* smem, const int h, const int n, const int cg, const int* st) {
  constexpr int NW = NT / 32;
  __shared__ float red_f[NW];
  __shared__ double red_d[NW];
  const int hd = p.hd, per = hd >> 5;
  // Everything up to pdl_wait() reads only what earlier steps left behind (device state, RoPE table, cached K/V rows of
  // older positions): it overlaps the tail of the QKV kernel.  q/k/v of this token are read after the wait.
  const int pos = st[1];                 // st = {token, position, step, n_total} of query token n
  if (pos >= p.n_ctx) return;
  const int T = pos + 1;
  const int n_total = max(T, min(st[3], p.n_ctx));
  const int n_vec = n_total & ~31;
  const int group = p.n_head / p.n_kv, kvh = h / group;
  const bool kv_writer = (h % group) == 0;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cp = kv_ctx_pad(p.n_ctx);

  float* sc = (float*)smem;                             // [cp] scores, then exp values
  uint16_t* p16 = (uint16_t*)(smem + (size_t)cp * 4);   // [cp] f16 probabilities, V-permuted order
  uint16_t* q16 = p16 + cp;                             // [hd] f16 rotated query, K-permuted order
  uint16_t* k16 = q16 + hd;                             // [hd] f16 rotated key of this position, K-permuted order
  uint16_t* v16 = k16 + hd;                             // [hd] f16 value of this position, natural order

  const int lim = min(T, n_vec);
  const uint16_t* vhead = p.vc + (size_t)kvh * hd * cp;
  constexpr int CPW = (ATTN_CH + NW - 1) / NW;          // V channels per warp (the last round may be partial)
  uint4 vpre[CPW][2];                                   // this warp's V rows, first two 256-position chunks
  uint2 kpre[8];                                        // this warp's first 8 K rows (hd == 128)
  float2 cs_pre = make_float2(1.f, 0.f);
#pragma unroll
  for (int j = 0; j < CPW; j++)
#pragma unroll
    for (int ch = 0; ch < 2; ch++)
      vpre[j][ch] = (ch * 256 < lim && warp + j * NW < ATTN_CH) ? *(const uint4*)(vhead + (size_t)(cg * ATTN_CH + warp + j * NW) * cp + ch * 256 + lane * 8) : make_uint4(0, 0, 0, 0);
  if (per == 4) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int t = min(warp * 8 + i, T - 1);
      kpre[i] = (t == pos) ? make_uint2(0, 0) : *(const uint2*)(p.kc + k_row(kvh, t, p.n_ctx, hd) + lane * 4);
    }
  } else if (per == 2) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int t = min(warp * 8 + i, T - 1);
      kpre[i] = make_uint2((t == pos) ? 0u : *(const uint32_t*)(p.kc + k_row(kvh, t, p.n_ctx, hd) + lane * 2), 0u);
    }
  }
  if (threadIdx.x < hd / 2) cs_pre = p.rope[(size_t)pos * (hd / 2) + threadIdx.x];
  if (PDLWAIT) pdl_wait();

  {  // RoPE (pairs) + f16 conversion of q, k, v for this position
    const float* qv = p.q + (size_t)n * p.q_stride + (size_t)h * hd;
    const float* kv = p.k + (size_t)n * p.kv_stride + (size_t)kvh * hd;
    const float* vv = p.v + (size_t)n * p.kv_stride + (size_t)kvh * hd;
    uint16_t* kd = p.kc + k_row(kvh, pos, p.n_ctx, hd);
    for (int i = threadIdx.x; i < hd / 2; i += NT) {
      const float2 cs = i == (int)threadIdx.x ? cs_pre : p.rope[(size_t)pos * (hd / 2) + i];
      const int i0 = p.neox ? i : 2 * i, i1 = p.neox ? i + hd / 2 : 2 * i + 1;
      float o0, o1;
      rope_pair(__ldcg(qv + i0), __ldcg(qv + i1), cs, p.neox, o0, o1);
      q16[k_perm(i0, hd)] = f2h(o0); q16[k_perm(i1, hd)] = f2h(o1);
      rope_pair(__ldcg(kv + i0), __ldcg(kv + i1), cs, p.neox, o0, o1);
      const uint16_t h0 = f2h(o0), h1 = f2h(o1);
      k16[k_perm(i0, hd)] = h0; k16[k_perm(i1, hd)] = h1;
      if (kv_writer && cg == 0) { kd[k_perm(i0, hd)] = h0; kd[k_perm(i1, hd)] = h1; }
    }
    for (int c = threadIdx.x; c < hd; c += NT) {
      const uint16_t hv = f2h(__ldcg(vv + c));
      v16[c] = hv;
      if (kv_writer && c / ATTN_CH == cg) p.vc[((size_t)kvh * hd + c) * cp + v_perm(pos)] = hv;
    }
  }
  attn_bar<BAR, NT>();

  if (per == 4) {
    // 8 cached rows per warp step, all loads issued before the first is used (the loop is latency-bound otherwise)
    const uint2 qq = *(const uint2*)(q16 + lane * 4);
    const float q0 = h2f((uint16_t)(qq.x & 0xffff)), q1 = h2f((uint16_t)(qq.x >> 16)), q2 = h2f((uint16_t)(qq.y & 0xffff)), q3 = h2f((uint16_t)(qq.y >> 16));
    for (int t0 = warp * 8; t0 < T; t0 += NW * 8) {
      uint2 kk[8];
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int t = min(t0 + i, T - 1);
        if (t == pos) kk[i] = *(const uint2*)(k16 + lane * 4);
        else if (t0 == warp * 8) kk[i] = kpre[i];
        else kk[i] = *(const uint2*)(p.kc + k_row(kvh, t, p.n_ctx, hd) + lane * 4);
      }
#pragma unroll
      for (int i = 0; i < 8; i++) {
        float s = 0.f;
        s = __fmaf_rn(h2f((uint16_t)(kk[i].x & 0xffff)), q0, s);
        s = __fmaf_rn(h2f((uint16_t)(kk[i].x >> 16)), q1, s);
        s = __fmaf_rn(h2f((uint16_t)(kk[i].y & 0xffff)), q2, s);
        s = __fmaf_rn(h2f((uint16_t)(kk[i].y >> 16)), q3, s);
        s = attn_reduce_f32x8(s);
        if (lane == 0 && t0 + i < T) sc[t0 + i] = __fmul_rn(s, p.kq_scale);
      }
    }
  } else if (per == 2) {
    // head_dim 64 (Falcon): the same 8-rows-in-flight scheme with 4-byte row pieces
    const uint32_t qq = *(const uint32_t*)(q16 + lane * 2);
    const float q0 = h2f((uint16_t)(qq & 0xffff)), q1 = h2f((uint16_t)(qq >> 16));
    for (int t0 = warp * 8; t0 < T; t0 += NW * 8) {
      uint32_t kk[8];
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int t = min(t0 + i, T - 1);
        if (t == pos) kk[i] = *(const uint32_t*)(k16 + lane * 2);
        else if (t0 == warp * 8) kk[i] = kpre[i].x;
        else kk[i] = *(const uint32_t*)(p.kc + k_row(kvh, t, p.n_ctx, hd) + lane * 2);
      }
#pragma unroll
      for (int i = 0; i < 8; i++) {
        float s = 0.f;
        s = __fmaf_rn(h2f((uint16_t)(kk[i] & 0xffff)), q0, s);
        s = __fmaf_rn(h2f((uint16_t)(kk[i] >> 16)), q1, s);
        s = attn_reduce_f32x8(s);
        if (lane == 0 && t0 + i < T) sc[t0 + i] = __fmul_rn(s, p.kq_scale);
      }
    }
  } else {
    for (int t = warp; t < T; t += NW) {
      const uint16_t* kr = (t == pos) ? (k16 + lane * per) : (p.kc + k_row(kvh, t, p.n_ctx, hd) + lane * per);
      float s = 0.f;
      for (int i = 0; i < per; i++) s = __fmaf_rn(h2f(kr[i]), h2f(q16[lane * per + i]), s);
      s = attn_reduce_f32x8(s);
      if (lane == 0) sc[t] = __fmul_rn(s, p.kq_scale);
    }
  }
  attn_bar<BAR, NT>();

  float mx = -INFINITY;
  for (int t = threadIdx.x; t < T; t += NT) mx = fmaxf(mx, sc[t]);
  mx = warp_max(mx);
  if (lane == 0) red_f[warp] = mx;
  attn_bar<BAR, NT>();
  mx = red_f[0];
#pragma unroll
  for (int w = 1; w < NW; w++) mx = fmaxf(mx, red_f[w]);
  double sum = 0.0;
  for (int t = threadIdx.x; t < T; t += NT) {
    const float val = h2f(__ldg(p.exp_tab + f2h(__fsub_rn(sc[t], mx))));
    sc[t] = val;
    sum += (double)val;
  }
  sum = warp_sum(sum);
  if (lane == 0) red_d[warp] = sum;
  attn_bar<BAR, NT>();
  sum = 0.0;
#pragma unroll
  for (int w = 0; w < NW; w++) sum += red_d[w];
  const float inv = (float)(1.0 / sum);
  const int t_end = (T + 255) & ~255;
  for (int t = threadIdx.x; t < t_end; t += NT) p16[v_perm(t)] = t < T ? f2h(__fmul_rn(sc[t], inv)) : (uint16_t)0;
  attn_bar<BAR, NT>();

  // V·P for this CTA's channels.  lane part: positions t < min(T, n_vec); lane L takes t = 32i+L in increasing i.
  // leftover part (ggml.c:2415-2418): positions n_vec <= t < T are added one by one in double after the lane reduction.  They
  // are the row i_left of one 256-position chunk, i.e. element i_left of lanes 0..T-n_vec-1 of that chunk's 16-byte loads:
  // every lane forms its float product and the warp adds them in lane order through shuffles.
  const int n_left = T - n_vec;                       // <= 31; <= 0 when the eval chunk extends past this token
  const int ch_left = n_vec >> 8, i_left = (n_vec & 255) >> 5;
#pragma unroll
  for (int j = 0; j < CPW; j++) {
    const int cc = warp + j * NW;
    if (cc >= ATTN_CH) break;
    const int c = cg * ATTN_CH + cc;
    const uint16_t* vrow = vhead + (size_t)c * cp;
    const uint16_t vcur = v16[c];
    float s = 0.f;
    for (int ch = 0; ch * 256 < lim; ch++) {
      uint4 vv;
      if (ch == 0) vv = vpre[j][0];
      else if (ch == 1) vv = vpre[j][1];
      else vv = *(const uint4*)(vrow + ch * 256 + lane * 8);
      const uint4 pp = *(const uint4*)(p16 + ch * 256 + lane * 8);
      const uint32_t vw[4] = {vv.x, vv.y, vv.z, vv.w}, pw[4] = {pp.x, pp.y, pp.z, pp.w};
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int t = ch * 256 + 32 * i + lane;
        if (t < lim) {
          uint16_t vh = (uint16_t)((vw[i >> 1] >> ((i & 1) * 16)) & 0xffff);
          const uint16_t ph = (uint16_t)((pw[i >> 1] >> ((i & 1) * 16)) & 0xffff);
          if (t == pos) vh = vcur;
          s = __fmaf_rn(h2f(vh), h2f(ph), s);
        }
      }
    }
    s = attn_reduce_f32x8(s);
    double sumf = (double)s;
    if (n_left > 0) {
      const int t = n_vec + lane;
      uint16_t vh = vrow[ch_left * 256 + lane * 8 + i_left];
      const uint16_t ph = p16[ch_left * 256 + lane * 8 + i_left];
      if (t == pos) vh = vcur;
      const float term = __fmul_rn(h2f(vh), h2f(ph));
      for (int l = 0; l < n_left; l++) sumf += (double)__shfl_sync(0xffffffffu, term, l);
    }
    if (lane == 0) p.out[(size_t)n * p.n_head * hd + (size_t)h * hd + c] = (float)sumf;
  }
}

static __global__ void __launch_bounds__(ATTN_THREADS) k_attn(const AttnParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  pdl_trigger();
  attn_body<ATTN_THREADS, 0, true>(p, smem, blockIdx.x, blockIdx.y, blockIdx.z, p.state);
}

// ----------------------------------------------------------------------------------------- argmax
// single block; writes the id of the largest logit (lowest id on ties) to out[0] and the number of logits equal to it to out[1]
static __global__ void k_argmax(const float* logits, int n, int* out) {
  __shared__ float bv[32];
  __shared__ int bi[32];
  __shared__ int ties;
  float best = -INFINITY;
  int idx = 0x7fffffff;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = logits[i];
    if (v > best) { best = v; idx = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > best || (ov == best && oi < idx)) { best = ov; idx = oi; }
  }
  if ((threadIdx.x & 31) == 0) { bv[threadIdx.x >> 5] = best; bi[threadIdx.x >> 5] = idx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); w++)
      if (bv[w] > best || (bv[w] == best && bi[w] < idx)) { best = bv[w]; idx = bi[w]; }
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
