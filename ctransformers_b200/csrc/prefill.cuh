// Batched prefill: up to PB_T = 32 prompt tokens per launch through the whole model, weights streamed ONCE per launch, the
// mat-muls as dense int8 tensor-core contractions — and every result identical, bit for bit, to the single-token path
// (and therefore to the reference's ggml_compute_forward_mul_mat with N columns, ggml.c:11031-11245, whose vec_dot treats
// every activation column on its own).
//
// The exact formulation.  Per (weight row, token, 256-block) the reference's AVX2 kernels need the eight int32 lane values
//     sumi[l] = Σ_s scale_s · Σ_{e<4} w[32s + 4l + e] · q8[32s + 4l + e]        (k_quants.c:1950-2052, 2651-2714, 3174-3262, 3794-3872)
// i.e. for a FIXED lane l a contraction over 32 (s, e) pairs — exactly the K = 32 of mma.sync.m16n8k32 — if the scale can
// ride on the weight operand.  w·scale does not fit a byte (15·63, 31·63, (q6-32)·int8, (q3-4)·(-32)), so it is split into two
// exact digits:  Q4_K / Q5_K: scale = 8·hi + lo (hi, lo <= 7; w·7 <= 217 fits u8)  →  sumi = D(w·lo) + 8·D(w·hi)
//                Q6_K / Q3_K: v = (q-32)·scale or (q-4)·(sc-32), v = 128·(v >> 7) + (v & 127)  →  sumi = D(v & 127) + 128·D(v >> 7)
// Two dense mma per (16 rows x 8 tokens x lane l x block): A = digits of 16 rows x 32 (s,e), B = int8 activations of 8 tokens,
// D = exact int32.  The fp32 part is the reference's: one fmadd per block into the lane accumulator, blocks in order,
// hsum_float_8 at the end (+ the mins accumulators) — the same instructions as stream.cuh, so the bits agree.
//
// Kernel structure = stream.cuh's (persistent CTAs, TMA weight ring, grid barriers), with phases over PB_T tokens:
//   QUANT   norm + Q8_K quantization of the PB_T activation vectors, ONE token per CTA (not redundantly in every CTA), written to
//           an L2-resident buffer in mma-B-fragment order
//   GEMM    consumer TEAMS of 4 warps own 16-row tiles; warp lp of a team owns AVX lanes 2lp, 2lp+1 (and mins lane lp) for all
//           32 tokens, keeps those accumulators in registers across the K loop, rebuilds its A digits once per block and
//           re-uses them for the 4 token groups; the team combines through shared memory at the end of a tile
//   KV      RoPE + fp16 store of K and V of all tokens (llama.cpp:2303-2335) — before any attention task reads the cache
//   ATTN    attention of every (token, head), one WARP per task (pb_attn_warp_task: the attention helpers of attention.cuh)
#pragma once
#include "stream.cuh"

namespace ctb {

constexpr int PB_T = 32;                   // tokens per launch
constexpr int PB_TG = PB_T / 8;            // token groups of 8 (mma N)
constexpr int PB_TEAMS = 2;
constexpr int PB_W = PB_TEAMS * 4;         // consumer warps
constexpr int PB_NT = PB_W * 32;
constexpr int PB_THREADS = PB_NT + 32;     // + producer warp
constexpr int PB_BAR = 1;                  // all consumers; team barriers: 2 + team
constexpr int PB_XCH = 12 * 16 * PB_T * 4; // bytes of a team's exchange buffer: (8 lanes + 4 mins) x 16 rows x PB_T tokens

enum : int { PP_EMBED = 0, PP_QUANT = 1, PP_GEMM = 2, PP_KV = 3, PP_ATTN = 4 };

// bytes of the quantized-activation buffer of a K-wide vector set: B fragments, mins pairs, block scales
__host__ __device__ inline size_t pb_qbuf_bytes(int K) { return (size_t)(K / 256) * (8192 + 512 + 128); }

struct alignas(16) PPhase {
  int kind;
  MVParams mv;            // QUANT: x, x2, x_mode, norm_*, eps, K;  GEMM: K, nseg, seg[], tables
  int x_ld, x2_ld;        // QUANT: floats between the token rows of x / x2
  int out_ld[MV_MAX_SEG], res_ld[MV_MAX_SEG], res2_ld[MV_MAX_SEG];   // GEMM: floats between token rows
  uint8_t* qbuf;          // QUANT writes, GEMM reads
  AttnParams at;          // KV / ATTN: q, k, v = rows of token 0, strides q_stride / kv_stride; out row stride n_head*hd
  EmbedParams em;         // EMBED: out row stride = K
  const int* state;       // [PB_T][4]: {token, position, step, n_total} per token; state[PB_T*4] = valid tokens of this launch
};
// Multi-sequence launches (the MS builds of k_pstep): the KV cache holds one region per sequence slot, and state[PB_S + i] is
// token i's slot.  state[PB_T*4 + 1] / [PB_T*4 + 2]: halves between the slots' K / V regions.
constexpr int PB_S = PB_T * 4 + 4;
constexpr int PB_STATE_MS = PB_S + PB_T;   // ints of a multi-sequence launch's state
__device__ __forceinline__ size_t pb_slot_off(const int* state, int tok, int which) { return (size_t)state[PB_S + tok] * (unsigned)state[PB_T * 4 + 1 + which]; }

struct PStepArgs {
  const PPhase* prog;
  int n_phases;
  int n_slots;
  unsigned* sync;
};

// ---------------------------------------------------------------------------------------------
// QUANT: the Q8_K image of one token (shared-memory layout of stage_activation) → global, in the order the GEMM warps load it
//   B     [b][tg][lp][lane = g*4+t][4 words]: (s=t, l=2lp) (s=t+4, l=2lp) (s=t, l=2lp+1) (s=t+4, l=2lp+1) of token tg*8+g
//   pairs [b][tg][k][token in group]  (stream.cuh StAct::pairs)       yd [b][token]
template <int NT, int BAR>
__device__ __forceinline__ void pb_quant_store(const uint8_t* smem, int K, int tok, uint8_t* qbuf) {
  const ActView a = act_view(ACT_Q8_K, K, const_cast<uint8_t*>(smem));
  const int nb = K >> 8, tg = tok >> 3, g = tok & 7;
  uint32_t* B = (uint32_t*)qbuf;
  uint32_t* pairs = (uint32_t*)(qbuf + (size_t)nb * 8192);
  float* yd = (float*)(qbuf + (size_t)nb * (8192 + 512));
  for (int i = threadIdx.x; i < nb * 64; i += NT) {
    const int b = i >> 6, s = (i >> 3) & 7, l = i & 7;
    const uint32_t w = *(const uint32_t*)(a.qs + q8k_word_offset(b, s, l));
    B[(((b * PB_TG + tg) * 4 + (l >> 1)) * 32 + g * 4 + (s & 3)) * 4 + (l & 1) * 2 + (s >> 2)] = w;
  }
  for (int i = threadIdx.x; i < nb * 4; i += NT) {
    const int b = i >> 2, k = i & 3;
    const int16_t* b4 = a.bs + b * 16 + 4 * k;
    const int p0 = (int)b4[0] + (int)b4[1], p1 = (int)b4[2] + (int)b4[3];
    pairs[((b * PB_TG + tg) * 4 + k) * 8 + g] = (uint32_t)(p0 & 0xffff) | ((uint32_t)p1 << 16);
  }
  for (int b = threadIdx.x; b < nb; b += NT) yd[b * PB_T + tok] = a.d[b];
  bar_sync<BAR, NT>();
}

// ---------------------------------------------------------------------------------------------
// GEMM consumer.  Warp lp of a team: AVX lanes l = 2lp + li (li = 0, 1).  Thread (g, t) of the warp holds, per token group tg,
//   acc[tg][li][r]  r = 0..3: (row g, token 8tg+2t) (row g, 8tg+2t+1) (row g+8, 8tg+2t) (row g+8, 8tg+2t+1)   — the mma D layout
//   am[tg][r]       the mins accumulator: Q4_K lane k = lp; Q5_K the scalar chain (warp lp == 0 only)
struct PBState { float acc[PB_TG][2][4]; float am[PB_TG][4]; };

__device__ __forceinline__ void mma_s8s8(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
      : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}

// weight word (row g+8rr, AVX lane l, word j) of a piece in the stream layout
__device__ __forceinline__ uint32_t pb_qs_word(const uint8_t* blk, int l, int rr, int g, int j) {
  return *(const uint32_t*)(blk + (((l >> 2) * 2 + rr) * 32 + g * 4 + (l & 3)) * 16 + j * 4);
}

template <int TYPE>
__device__ __forceinline__ void pb_block(const uint8_t* blk, int b, const uint8_t* qbuf, int nb, int lane, int lp, int ntg, PBState& st) {
  const int g = lane >> 2, t = lane & 3;
  const uint32_t* Bq = (const uint32_t*)qbuf;
  const uint32_t* pairs = (const uint32_t*)(qbuf + (size_t)nb * 8192);
  const float* ydp = (const float*)(qbuf + (size_t)nb * (8192 + 512));
  // ---- A digits of this warp's two AVX lanes: fragment register i = (sub-block s = t + 4(i>>1), row g + 8(i&1))
  uint32_t Alo[2][4], Ahi[2][4];
  float dw[2], dmin[2] = {0.f, 0.f};
  uint32_t mw[2] = {0u, 0u};          // Q4_K: the two mins bytes of lane k = lp, rows g / g+8
  uint32_t m03[2] = {0u, 0u}, m47[2] = {0u, 0u};
  if (TYPE == GT_Q4_K || TYPE == GT_Q5_K) {
    const int hoff = TYPE == GT_Q4_K ? 2048 : 2560;
    uint32_t slo[2][2], shi[2][2];   // [rr][s = t, t+4]
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
      const int4 h = ((const int4*)(blk + hoff))[rr * 8 + g];
      uint32_t sc03, sc47;
      unpack_k4((uint32_t)h.y, (uint32_t)h.z, (uint32_t)h.w, sc03, sc47, m03[rr], m47[rr]);
      const uint32_t s0 = (sc03 >> (8 * t)) & 0xffu, s1 = (sc47 >> (8 * t)) & 0xffu;
      slo[rr][0] = s0 & 7u; shi[rr][0] = s0 >> 3; slo[rr][1] = s1 & 7u; shi[rr][1] = s1 >> 3;
      dw[rr] = h2f((uint16_t)((uint32_t)h.x & 0xffffu));
      dmin[rr] = h2f((uint16_t)((uint32_t)h.x >> 16));
      mw[rr] = (lp < 2 ? m03[rr] : m47[rr]) >> ((lp & 1) * 16);
    }
#pragma unroll
    for (int li = 0; li < 2; li++) {
      const int l = 2 * lp + li;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int rr = i & 1, hs = i >> 1;                 // sub-block s = t + 4hs = 2j + (t & 1), j = (t >> 1) + 2hs
        const uint32_t w = pb_qs_word(blk, l, rr, g, (t >> 1) + 2 * hs);
        uint32_t q = (w >> (4 * (t & 1))) & 0x0f0f0f0fu;
        if (TYPE == GT_Q5_K) {                              // bit s of a qh byte: 5th bit of the element in sub-block s
          const uint32_t hb = *(const uint32_t*)(blk + 2048 + (((l >> 2) * 2 + rr) * 32 + g * 4 + (l & 3)) * 4);
          q |= ((hb >> (t + 4 * hs)) & 0x01010101u) << 4;
        }
        Alo[li][i] = q * slo[rr][hs];                       // per byte <= 31·7: no carry between bytes
        Ahi[li][i] = q * shi[rr][hs];
      }
    }
  } else if (TYPE == GT_Q3_K) {   // v = (q3 - 4)·(sc - 32) in [-124, 128], split as Q6_K's
    const uint32_t* sp = (const uint32_t*)(blk + 1536);
    dw[0] = h2f(((const uint16_t*)(blk + 1728))[g]);
    dw[1] = h2f(((const uint16_t*)(blk + 1728))[8 + g]);
    const int par = lp >> 1;   // both lanes l = 2lp + li lie in the same 16-weight half of each group
    int sc[2][2];              // [rr][hs]: the six-bit scale of sub-block 2·grp + par, grp = t + 4hs (k_quants.c:1968-1974)
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
      const uint32_t* h = sp + 3 * (rr * 8 + g);
      const uint32_t a0 = h[0], a1 = h[1], a2 = h[2];
      const uint32_t lo = (t >> 1) ? a1 : a0;   // sub-blocks 2t + par (word t >> 1) and 8 + 2t + par (word 2 + (t >> 1))
      const int byte = 2 * (t & 1) + par, sh = 8 * byte;
      sc[rr][0] = (int)(((lo >> sh) & 0x0fu) | (((a2 >> (sh + 2 * (t >> 1))) & 0x03u) << 4)) - 32;
      sc[rr][1] = (int)(((lo >> (sh + 4)) & 0x0fu) | (((a2 >> (sh + 4 + 2 * (t >> 1))) & 0x03u) << 4)) - 32;
    }
#pragma unroll
    for (int li = 0; li < 2; li++) {
      const int l = 2 * lp + li;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int rr = i & 1, hs = i >> 1, grp = t + 4 * hs;   // qs word hs, bits 2t; hmask bit grp
        const int e0 = (((l >> 2) * 2 + rr) * 32 + g * 4 + (l & 3));
        const uint32_t qw = *(const uint32_t*)(blk + e0 * 8 + hs * 4);
        const uint32_t hm = *(const uint32_t*)(blk + 1024 + e0 * 4);
        const uint32_t u = ((qw >> (2 * t)) & 0x03030303u) | (((hm >> grp) & 0x01010101u) << 2);
        const int scale = sc[rr][hs];
        uint32_t lo = 0u, hi = 0u;
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const int v = ((int)((u >> (8 * e)) & 0xffu) - 4) * scale;
          lo |= (uint32_t)(v & 127) << (8 * e);
          hi |= (uint32_t)((v >> 7) & 0xff) << (8 * e);
        }
        Alo[li][i] = lo; Ahi[li][i] = hi;
      }
    }
  } else {   // Q6_K: v = (q6 - 32)·scale split into v >> 7 (signed) and v & 127
    const int4 s0 = ((const int4*)(blk + 3072))[g], s1 = ((const int4*)(blk + 3072))[8 + g];
    dw[0] = h2f(((const uint16_t*)(blk + 3328))[g]);
    dw[1] = h2f(((const uint16_t*)(blk + 3328))[8 + g]);
#pragma unroll
    for (int li = 0; li < 2; li++) {
      const int l = 2 * lp + li, par = l >> 2;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int rr = i & 1, jj = i >> 1;                  // 32-weight group grp = t + 4jj = jj*4 + m, m = t
        const uint32_t ql = pb_qs_word(blk, l, rr, g, jj * 2 + (t & 1));               // m odd: the second 32 bytes (v = 1)
        const uint32_t qh = *(const uint32_t*)(blk + 2048 + (((l >> 2) * 2 + rr) * 32 + g * 4 + (l & 3)) * 8 + jj * 4);
        const uint32_t u = ((ql >> (4 * (t >> 1))) & 0x0f0f0f0fu) | (((qh >> (2 * t)) & 0x03030303u) << 4);
        const int4 sv = rr ? s1 : s0;
        const uint32_t swd = jj ? (uint32_t)((t >> 1) ? sv.w : sv.z) : (uint32_t)((t >> 1) ? sv.y : sv.x);   // word jj*2 + (m >> 1)
        const int scale = (int)(int8_t)((swd >> (8 * (2 * (t & 1) + par))) & 0xffu);                          // byte 2(m & 1) + par
        uint32_t lo = 0u, hi = 0u;
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const int v = ((int)((u >> (8 * e)) & 0xffu) - 32) * scale;
          lo |= (uint32_t)(v & 127) << (8 * e);
          hi |= (uint32_t)((v >> 7) & 0xff) << (8 * e);
        }
        Alo[li][i] = lo; Ahi[li][i] = hi;
      }
    }
  }
  // ---- the four token groups
#pragma unroll
  for (int tg = 0; tg < PB_TG; tg++) {
    if (tg >= ntg) break;   // a short batch (the tail of a prompt) skips its empty token groups
    const uint4 bw = __ldg((const uint4*)(Bq + (size_t)(((b * PB_TG + tg) * 4 + lp) * 32 + lane) * 4));
    const float2 yd = __ldg((const float2*)(ydp + b * PB_T + tg * 8 + 2 * t));
    float dd[4], ddm[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const float y = (r & 1) ? yd.y : yd.x;
      dd[r] = __fmul_rn(y, dw[r >> 1]);
      ddm[r] = __fmul_rn(-y, dmin[r >> 1]);
    }
#pragma unroll
    for (int li = 0; li < 2; li++) {
      const uint32_t b0 = li ? bw.z : bw.x, b1 = li ? bw.w : bw.y;
      int Dl[4], Dh[4];
      if (TYPE == GT_Q6_K || TYPE == GT_Q3_K) {
        mma_s8s8(Dl, Alo[li][0], Alo[li][1], Alo[li][2], Alo[li][3], b0, b1);
        mma_s8s8(Dh, Ahi[li][0], Ahi[li][1], Ahi[li][2], Ahi[li][3], b0, b1);
      } else {
        mma_u8s8(Dl, Alo[li][0], Alo[li][1], Alo[li][2], Alo[li][3], b0, b1, 0, 0);
        mma_u8s8(Dh, Ahi[li][0], Ahi[li][1], Ahi[li][2], Ahi[li][3], b0, b1, 0, 0);
      }
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int sumi = Dl[r] + (TYPE == GT_Q6_K || TYPE == GT_Q3_K ? 128 : 8) * Dh[r];
        st.acc[tg][li][r] = __fmaf_rn(dd[r], (float)sumi, st.acc[tg][li][r]);
      }
    }
    if (TYPE == GT_Q4_K) {          // mins lane k = lp: m[2k]·(bsums[4k]+bsums[4k+1]) + m[2k+1]·(bsums[4k+2]+bsums[4k+3])
      const uint2 pw = __ldg((const uint2*)(pairs + ((b * PB_TG + tg) * 4 + lp) * 8 + 2 * t));
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int pm = __dp2a_lo((int)((r & 1) ? pw.y : pw.x), (int)mw[r >> 1], 0);
        st.am[tg][r] = __fmaf_rn(ddm[r], (float)pm, st.am[tg][r]);
      }
    } else if (TYPE == GT_Q5_K) {   // the scalar mins chain Σ_k m[k]·(bsums[2k]+bsums[2k+1]): kept by warp lp == 0
      if (lp == 0) {
        uint2 pk[4];
#pragma unroll
        for (int k = 0; k < 4; k++) pk[k] = __ldg((const uint2*)(pairs + ((b * PB_TG + tg) * 4 + k) * 8 + 2 * t));
#pragma unroll
        for (int r = 0; r < 4; r++) {
          const int rr = r >> 1;
          int hs = __dp2a_lo((int)((r & 1) ? pk[0].y : pk[0].x), (int)m03[rr], 0);
          hs = __dp2a_hi((int)((r & 1) ? pk[1].y : pk[1].x), (int)m03[rr], hs);
          hs = __dp2a_lo((int)((r & 1) ? pk[2].y : pk[2].x), (int)m47[rr], hs);
          hs = __dp2a_hi((int)((r & 1) ? pk[3].y : pk[3].x), (int)m47[rr], hs);
          st.am[tg][r] = __fmaf_rn(ddm[r], (float)hs, st.am[tg][r]);
        }
      }
    }
  }
}

template <int TYPE>
__device__ __forceinline__ void pb_chunk(const uint8_t* slot, int nblk, int b0, const uint8_t* qbuf, int nb, int lane, int lp, int ntg, PBState& st) {
  constexpr int BB = StTraits<TYPE>::BB;
#pragma unroll 1
  for (int i = 0; i < nblk; i++) pb_block<TYPE>(slot + i * BB, b0 + i, qbuf, nb, lane, lp, ntg, st);
}

// end of a tile: the team's 4 warps publish their accumulators, then its 128 threads finish 16 rows x PB_T tokens:
// hsum_float_8's tree over the 8 lanes (ggml.c:609-615), the mins tail, the epilogue (matvec.cuh) per token row
template <int BARID>
__device__ __forceinline__ void pb_finish(const PBState& st, float* xch, int type, int lane, int lp, int tid_team, const PPhase& ph, int n_tok, int seg, int row0) {
  const int g = lane >> 2, t = lane & 3;
  asm volatile("bar.sync %0, %1;" ::"n"(BARID), "n"(128) : "memory");   // the previous tile's readers are done with xch
#pragma unroll
  for (int tg = 0; tg < PB_TG; tg++)
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int row = g + 8 * (r >> 1), tok = tg * 8 + 2 * t + (r & 1);
#pragma unroll
      for (int li = 0; li < 2; li++) xch[((2 * lp + li) * 16 + row) * PB_T + tok] = st.acc[tg][li][r];
      if (type == GT_Q4_K || (type == GT_Q5_K && lp == 0)) xch[((8 + lp) * 16 + row) * PB_T + tok] = st.am[tg][r];
    }
  asm volatile("bar.sync %0, %1;" ::"n"(BARID), "n"(128) : "memory");
  const MVSeg& sg = ph.mv.seg[seg];
  const int old = ph.out_ld[seg], rld = ph.res_ld[seg], r2ld = ph.res2_ld[seg];
  for (int idx = tid_team; idx < 16 * PB_T; idx += 128) {
    const int row = idx & 15, tok = idx >> 4;
    const float* x = xch + row * PB_T + tok;
    constexpr int L = 16 * PB_T;
    float v = __fadd_rn(__fadd_rn(__fadd_rn(x[0 * L], x[4 * L]), __fadd_rn(x[2 * L], x[6 * L])),
                        __fadd_rn(__fadd_rn(x[1 * L], x[5 * L]), __fadd_rn(x[3 * L], x[7 * L])));
    if (type == GT_Q4_K) v = __fadd_rn(v, __fadd_rn(__fadd_rn(x[8 * L], x[10 * L]), __fadd_rn(x[9 * L], x[11 * L])));
    else if (type == GT_Q5_K) v = __fadd_rn(v, x[8 * L]);
    const int grow = row0 + row;
    if (grow < sg.w.M && tok < n_tok) sg.out[(size_t)tok * old + grow] = epilogue(sg.epi, v, sg.res + (size_t)tok * rld + grow, sg.res2 + (size_t)tok * r2ld + grow, ph.mv);
  }
}

// ---------------------------------------------------------------------------------------------
// Ring addressing: every team owns PB_TEAMS-strided slots of the ring (ring_pos in stream.cuh); cnt[t] counts team t's items.
template <bool Q3>
__device__ __forceinline__ void pb_producer(const PStepArgs& args, uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar) {
  const int lane = threadIdx.x & 31;
  const uint32_t D = (uint32_t)(args.n_slots / PB_TEAMS);
  uint32_t cnt[PB_TEAMS];
#pragma unroll
  for (int t = 0; t < PB_TEAMS; t++) cnt[t] = 0;
  for (int ip = 0; ip < args.n_phases; ip++) {
    const PPhase* ph = args.prog + ip;
    if (ph->kind != PP_GEMM) continue;
    const MVParams& p = ph->mv;
    TileSpace ts;
    ts.init<Q3>(p);
    const int T0 = ts.boundary(blockIdx.x, gridDim.x), T1 = ts.boundary(blockIdx.x + 1, gridDim.x);
    const int nb = p.K >> 8;
    for (int w0 = T0; w0 < T1; w0 += PB_TEAMS) {
      const int ntw = min(PB_TEAMS, T1 - w0);
      const TileInfo ti = tile_info<Q3>(ts, p, w0 + lane, nb, lane < ntw);
      for (int kc = 0;; kc++) {
        const unsigned mask = __ballot_sync(0xffffffffu, kc < ti.nch);
        if (!mask) break;
#pragma unroll
        for (int j = 0; j < PB_TEAMS; j++) {   // tile w0 + j belongs to team j
          if (!((mask >> j) & 1u)) continue;
          const int seg = __shfl_sync(0xffffffffu, ti.seg, j), til = __shfl_sync(0xffffffffu, ti.til, j), type = __shfl_sync(0xffffffffu, ti.type, j);
          if (lane == 0) {
            const RingPos rp = ring_pos(cnt[j], (uint32_t)j, PB_TEAMS, D);
            const StItem it = st_item<Q3>(p, seg, type, til, kc, nb);
            mbar_wait(&empty_bar[rp.slot], rp.parity ^ 1u, W_PF_FREE_SLOT, (int)cnt[j]);
            mbar_expect_tx(&full_bar[rp.slot], it.bytes);
            bulk_g2s(ring + (size_t)rp.slot * ST_SLOT, it.src, it.bytes, &full_bar[rp.slot]);
          }
          cnt[j]++;
        }
      }
    }
  }
}

template <bool Q3>
__device__ __forceinline__ void pb_gemm_phase(const PPhase& ph, int n_tok, uint8_t* ring, float* xch_all, uint64_t* full_bar, uint64_t* empty_bar, uint32_t D, uint32_t& cnt) {
  const MVParams& p = ph.mv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, team = warp >> 2, lp = warp & 3;
  float* xch = xch_all + (size_t)team * (PB_XCH / 4);
  TileSpace ts;
  ts.init<Q3>(p);
  const int T0 = ts.boundary(blockIdx.x, gridDim.x), T1 = ts.boundary(blockIdx.x + 1, gridDim.x);
  const int nb = p.K >> 8;
#pragma unroll 1
  for (int w0 = T0; w0 < T1; w0 += PB_TEAMS) {
    const int ntw = min(PB_TEAMS, T1 - w0);
    const TileInfo ti = tile_info<Q3>(ts, p, w0 + lane, nb, lane < ntw);
    const int my_seg = __shfl_sync(0xffffffffu, ti.seg, team), my_til = __shfl_sync(0xffffffffu, ti.til, team), my_type = __shfl_sync(0xffffffffu, ti.type, team);
    PBState st;
#pragma unroll
    for (int tg = 0; tg < PB_TG; tg++)
#pragma unroll
      for (int r = 0; r < 4; r++) { st.acc[tg][0][r] = 0.f; st.acc[tg][1][r] = 0.f; st.am[tg][r] = 0.f; }
#pragma unroll 1
    for (int kc = 0;; kc++) {
      const unsigned mask = __ballot_sync(0xffffffffu, kc < ti.nch);
      if (!mask) break;
      if ((mask >> team) & 1u) {
        const RingPos rp = ring_pos(cnt, (uint32_t)team, PB_TEAMS, D);
        const int kb = st_chunk_blocks<Q3>(my_type);
        const int b0 = kc * kb, nblk = min(kb, nb - b0);
        const uint8_t* sp = ring + (size_t)rp.slot * ST_SLOT;
        mbar_wait(&full_bar[rp.slot], rp.parity, W_PF_WEIGHT_ITEM, (int)cnt);
        if (my_type == GT_Q4_K) pb_chunk<GT_Q4_K>(sp, nblk, b0, ph.qbuf, nb, lane, lp, (n_tok + 7) >> 3, st);
        else if (my_type == GT_Q6_K) pb_chunk<GT_Q6_K>(sp, nblk, b0, ph.qbuf, nb, lane, lp, (n_tok + 7) >> 3, st);
        else if (Q3 && my_type == GT_Q3_K) pb_chunk<GT_Q3_K>(sp, nblk, b0, ph.qbuf, nb, lane, lp, (n_tok + 7) >> 3, st);
        else pb_chunk<GT_Q5_K>(sp, nblk, b0, ph.qbuf, nb, lane, lp, (n_tok + 7) >> 3, st);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[rp.slot]);   // 4 arrivals (the team's warps) free the slot
        cnt++;
      }
    }
    if (team < ntw) {
      if (team == 0) pb_finish<2>(st, xch, my_type, lane, lp, threadIdx.x & 127, ph, n_tok, my_seg, my_til * ST_ROWS);
      else pb_finish<3>(st, xch, my_type, lane, lp, threadIdx.x & 127, ph, n_tok, my_seg, my_til * ST_ROWS);
    }
  }
}

// RoPE of K + fp16 store of K and V of every valid token (attn_stage's cache writes, for the whole batch); MS: into its slot's region
template <bool MS>
__device__ __forceinline__ void pb_kv_phase(const PPhase& ph, int n_tok) {
  const AttnParams& a = ph.at;
  const int half = a.hd / 2, per_tok = a.n_kv * half, total = n_tok * per_tok;
  for (int idx = blockIdx.x * PB_NT + threadIdx.x; idx < total; idx += gridDim.x * PB_NT) {
    const int tok = idx / per_tok, r = idx % per_tok, kh = r / half, i = r % half;
    const int pos = ph.state[tok * 4 + 1];
    if (pos >= a.n_ctx) continue;
    if constexpr (MS) {
      uint16_t* kc = a.kc + pb_slot_off(ph.state, tok, 0);
      uint16_t* vc = a.vc + pb_slot_off(ph.state, tok, 1);
      rope_k_pair(a.k + (size_t)tok * a.kv_stride + (size_t)kh * a.hd, i, a.hd, a.neox, a.rope[(size_t)pos * half + i], kc + k_row(kh, pos, a.n_ctx, a.hd));
      const float* vsrc = a.v + (size_t)tok * a.kv_stride + (size_t)kh * a.hd;
      for (int c = 2 * i; c < 2 * i + 2; c++) vc[v_chan(kh, c, a.n_ctx, a.hd) + v_perm(pos)] = f2h(__ldcg(vsrc + c));
    } else {   // (kept as it was: one expression for both builds changes the instructions ptxas emits for this one)
      rope_k_pair(a.k + (size_t)tok * a.kv_stride + (size_t)kh * a.hd, i, a.hd, a.neox, a.rope[(size_t)pos * half + i], a.kc + k_row(kh, pos, a.n_ctx, a.hd));
      const float* vsrc = a.v + (size_t)tok * a.kv_stride + (size_t)kh * a.hd;
      for (int c = 2 * i; c < 2 * i + 2; c++) a.vc[v_chan(kh, c, a.n_ctx, a.hd) + v_perm(pos)] = f2h(__ldcg(vsrc + c));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Attention of one (token, head) by ONE warp (the CTA-wide attn_body of the decode path is a latency chain per task; a prompt
// batch has n_tok x n_head independent tasks, so here every warp takes its own): the attention helpers of attention.cuh with
// NT = 32.  K and V of every position — the token's own included — come from the cache: the KV phase has stored the whole
// batch before any task starts.
__host__ __device__ inline size_t pb_attn_warp_bytes(int n_ctx, int hd) { return (attn_scratch(nullptr, n_ctx, hd, false).bytes + 15) & ~(size_t)15; }

template <bool GEN>
__device__ __forceinline__ void pb_attn_warp_task(const AttnParams& p, const int* st, int tok, int h, uint8_t* wsm) {
  const AttnPos a = attn_pos(p, st);
  if (a.T == 0) return;
  const int hd = p.hd, kvh = h / (p.n_head / p.n_kv), lane = threadIdx.x & 31;
  const AttnScratch s = attn_scratch<GEN>(wsm, p.n_ctx, hd, false);
  attn_stage<32, GEN>(p, s, tok, h, 0, a.pos, attn_cs0<32>(p, a.pos));
  __syncwarp();
  attn_scores<GEN>(hd, p.kc + k_row<GEN>(kvh, 0, p.n_ctx, hd), a.T, 0, 8, s.q16, p.kq_scale, s.sc);
  __syncwarp();
  attn_softmax<32, 0>(s.sc, s.p16, a.T, p.exp_tab, nullptr, nullptr);
  float* orow = p.out + (size_t)tok * p.n_head * hd + (size_t)h * hd;
  for (int c = 0; c < hd; c++) {
    const float o = attn_vp(p.vc + v_chan(kvh, c, p.n_ctx, hd), s.p16, a, -1, 0);
    if (lane == 0) orow[c] = o;
  }
  __syncwarp();
}

// the ATTN phase of one CTA's warp: hd 64 / 128 inline, other head sizes in one out-of-line call; MS: each token reads its
// slot's region of the cache
template <bool GEN, bool MS>
__device__ __forceinline__ void pb_attn_phase(const PPhase& ph, int n_tok, uint8_t* work) {
  const int warp = threadIdx.x >> 5;
  const int n_tasks = n_tok * ph.at.n_head;
  uint8_t* wsm = work + (size_t)warp * pb_attn_warp_bytes(ph.at.n_ctx, ph.at.hd);
  for (int task = blockIdx.x * PB_W + warp; task < n_tasks; task += (int)gridDim.x * PB_W) {
    const int tok = task / ph.at.n_head;
    if constexpr (MS) {
      AttnParams p = ph.at;
      p.kc += pb_slot_off(ph.state, tok, 0);
      p.vc += pb_slot_off(ph.state, tok, 1);
      pb_attn_warp_task<GEN>(p, ph.state + tok * 4, tok, task % ph.at.n_head, wsm);
    } else {
      pb_attn_warp_task<GEN>(ph.at, ph.state + tok * 4, tok, task % ph.at.n_head, wsm);
    }
  }
}
// (one copy per kernel build, Q3 / MS: ptxas fits an out-of-line function's registers to all its callers at once)
template <bool Q3, bool MS>
static __device__ __noinline__ void pb_attn_phase_gen(const PPhase& ph, int n_tok, uint8_t* work) { pb_attn_phase<true, MS>(ph, n_tok, work); }

// Q3: the build for programs that hold Q3_K matrices or a Q3_K embedding table.  The build without it compiles to the same
// instructions as before Q3_K was added; with the Q3_K code inlined into the one kernel, ptxas spilled more there (DESIGN.md §6).
// MS: the build for multi-sequence launches (a KV slot per token, PB_S), kept apart for the same reason: the single-sequence
// builds compile to the same instructions as before it was added.  A QUANT phase with norm_out set (the output head's) also
// writes every token's normalised row there, norm_out + token * K (the embeddings).
template <bool Q3, bool MS = false>
static __global__ void __launch_bounds__(PB_THREADS, 1) k_pstep(const __grid_constant__ PStepArgs args) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ __align__(8) uint64_t full_bar[ST_MAX_SLOTS];
  __shared__ __align__(8) uint64_t empty_bar[ST_MAX_SLOTS];
  __shared__ double red[3 * PB_W];
  __shared__ __align__(16) PPhase ph;
  const int warp = threadIdx.x >> 5;
  uint8_t* ring = smem;
  uint8_t* work = smem + (size_t)args.n_slots * ST_SLOT;   // activation image (QUANT) / team exchange buffers (GEMM) / attention scratch
  ring_init(full_bar, empty_bar, args.n_slots, 4);
  if (warp == PB_W) {
    pb_producer<Q3>(args, ring, full_bar, empty_bar);
    return;
  }
  const unsigned G = gridDim.x;
  uint32_t seq = 0;   // this warp's team's item count
#pragma unroll 1
  for (int ip = 0; ip < args.n_phases; ip++) {
    bar_sync<PB_BAR, PB_NT>();
    if (threadIdx.x == 0 && ip > 0) { __threadfence(); atomicAdd(args.sync, 1u); }
    {
      const uint4* src = (const uint4*)(args.prog + ip);
      uint4* dst = (uint4*)&ph;
      for (int i = threadIdx.x - 32; i >= 0 && i < (int)(sizeof(PPhase) / 16); i += PB_NT - 32) dst[i] = __ldg(src + i);
    }
    bar_sync<PB_BAR, PB_NT>();
    if (threadIdx.x == 0 && ip > 0) {
      const unsigned target = (unsigned)ip * G;
      bounded_wait([&] { return ld_acquire_u32(args.sync) >= target; }, W_PF_GRID_BARRIER, ip);
    }
    bar_sync<PB_BAR, PB_NT>();
    const int n_tok = min(PB_T, ph.state[PB_T * 4]);
    if (ph.kind == PP_GEMM) {
      pb_gemm_phase<Q3>(ph, n_tok, ring, (float*)work, full_bar, empty_bar, (uint32_t)(args.n_slots / PB_TEAMS), seq);
    } else if (ph.kind == PP_QUANT) {
      for (int tok = blockIdx.x; tok < n_tok; tok += G) {
        MVParams q = ph.mv;
        q.x = ph.mv.x + (size_t)tok * ph.x_ld;
        if (q.x2) q.x2 = ph.mv.x2 + (size_t)tok * ph.x2_ld;
        if constexpr (MS) {
          if (q.norm_out) q.norm_out = ph.mv.norm_out + (size_t)tok * q.K;
        }
        NormPre np;
        preload_norm(np, q);
        if constexpr (MS) stage_activation<PB_NT, PB_BAR>(q, np, ACT_Q8_K, work, red, q.norm_out != nullptr);
        else stage_activation<PB_NT, PB_BAR>(q, np, ACT_Q8_K, work, red, false);
        pb_quant_store<PB_NT, PB_BAR>(work, q.K, tok, ph.qbuf);
      }
    } else if (ph.kind == PP_KV) {
      pb_kv_phase<MS>(ph, n_tok);
    } else if (ph.kind == PP_ATTN) {
      if (attn_fast_hd(ph.at.hd)) pb_attn_phase<false, MS>(ph, n_tok, work);
      else pb_attn_phase_gen<Q3, MS>(ph, n_tok, work);
    } else if (ph.kind == PP_EMBED) {
      for (int tok = blockIdx.x; tok < n_tok; tok += G) embed_row<Q3>(ph.em, ph.state[tok * 4], ph.em.out + (size_t)tok * ph.em.K, threadIdx.x, PB_NT);
    }
  }
  bar_sync<PB_BAR, PB_NT>();
  grid_rearm(args.sync);
}

// ---------------------------------------------------------------------------------------------
// Host side
inline size_t pb_work_bytes(int K_max, int n_ctx, int hd) {
  size_t w = std::max<size_t>((size_t)PB_TEAMS * PB_XCH, act_smem_bytes(ACT_Q8_K, K_max) + 64);
  w = std::max(w, (size_t)PB_W * pb_attn_warp_bytes(n_ctx, hd));
  return (w + 127) & ~(size_t)127;
}
// launch shape of k_pstep around `work` bytes of scratch: whole per-team sub-rings in what shared memory has left.  false
// when fewer than 4 slots fit (the attention scratch of a long context): the caller then has no batched prefill.
inline bool pstep_shape(size_t work, int& n_slots, size_t& smem) {
  const size_t room = std::min(std::min(max_dyn_smem(k_pstep<false>), max_dyn_smem(k_pstep<true>)),
                               std::min(max_dyn_smem(k_pstep<false, true>), max_dyn_smem(k_pstep<true, true>)));
  if (work + 4 * (size_t)ST_SLOT > room) return false;
  n_slots = (int)std::min<size_t>(ST_MAX_SLOTS, (room - work) / ST_SLOT) / PB_TEAMS * PB_TEAMS;
  smem = (size_t)n_slots * ST_SLOT + work;
  return true;
}
// The QUANT + GEMM phase pair of one mat-vec m over PB_T-token buffers.  bat(p, ld) maps each activation pointer of m (x, x2, a
// segment's out / res / res2) to its PB_T-row buffer and sets ld to the floats between token rows (null: null, 0).  qbuf holds
// pb_qbuf_bytes(m.K), one per pair: nothing stale of another phase can sit in an L1.
template <typename Bat>
inline void pb_matvec_phases(const MVParams& m, uint8_t* qbuf, const int* state, Bat&& bat, std::vector<PPhase>& prog) {
  PPhase ph{};
  ph.state = state;
  ph.mv = m;
  ph.mv.norm_out = nullptr;
  ph.mv.x = bat(m.x, ph.x_ld);
  ph.mv.x2 = bat(m.x2, ph.x2_ld);
  ph.qbuf = qbuf;
  ph.kind = PP_QUANT; prog.push_back(ph);
  for (int s = 0; s < m.nseg; s++) {
    ph.mv.seg[s].out = bat(m.seg[s].out, ph.out_ld[s]);
    ph.mv.seg[s].res = bat(m.seg[s].res, ph.res_ld[s]);
    ph.mv.seg[s].res2 = bat(m.seg[s].res2, ph.res2_ld[s]);
  }
  ph.kind = PP_GEMM; prog.push_back(ph);
}
static inline cudaError_t pstep_set_smem_limit(size_t bytes) {
  for (auto k : {k_pstep<false>, k_pstep<true>, k_pstep<false, true>, k_pstep<true, true>}) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}
// does a program hold Q3_K matrices or a Q3_K embedding table (then it runs on k_pstep<true>)?
inline bool pstep_q3(const std::vector<PPhase>& prog) {
  for (const PPhase& ph : prog) {
    if (ph.kind == PP_EMBED && ph.em.type == GT_Q3_K) return true;
    if (ph.kind == PP_GEMM)
      for (int s = 0; s < ph.mv.nseg; s++)
        if (ph.mv.seg[s].w.type == GT_Q3_K) return true;
  }
  return false;
}
static inline cudaError_t launch_pstep(int grid, int n_slots, size_t smem, cudaStream_t st, const PPhase* d_prog, int n_phases, unsigned* d_sync, bool q3 = false,
                                       bool ms = false) {
  PStepArgs a;
  a.prog = d_prog; a.n_phases = n_phases; a.n_slots = n_slots; a.sync = d_sync;
  if (ms) {
    if (q3) k_pstep<true, true><<<grid, PB_THREADS, smem, st>>>(a);
    else k_pstep<false, true><<<grid, PB_THREADS, smem, st>>>(a);
  } else if (q3) k_pstep<true><<<grid, PB_THREADS, smem, st>>>(a);
  else k_pstep<false><<<grid, PB_THREADS, smem, st>>>(a);
  return cudaGetLastError();
}

}  // namespace ctb
