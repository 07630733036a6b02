// The persistent decode-step kernel (sm_90a): every K-quant mat-vec of a token, plus attention, embedding row and greedy
// pick, as PHASES of one launch — one CTA per SM, device-side grid barriers instead of kernel boundaries, and a weight
// stream that never stops at them.
//
// Replaces, bit-exactly, what ggml_graph_compute does per token for a Llama / Falcon graph (llama.cpp:2162-2798, 2835-2981):
//   ggml_compute_forward_mul_mat over Q3_K / Q4_K / Q5_K / Q6_K weights with Q8_K activations   ggml.c:11031-11245
//   ggml_vec_dot_q3_K_q8_K / q4_K / q5_K / q6_K, AVX2 variants              k_quants.c:1950-2052, 2651-2714, 3174-3262, 3794-3872
//   norm + quantize prologue and residual / SiLU / GELU epilogue                         matvec.cuh (shared with k_matvec)
//   RoPE, KV store, K·q, softmax, V·p                                                    attention.cuh (attn_body, or st_attn_task below)
//
// Structure of a CTA (ST_W consumer warps + 1 producer warp):
//   producer warp   walks the phase list ahead of everybody else and keeps a ring of ST_SLOT-byte shared-memory slots full:
//                   one cp.async.bulk (TMA bulk copy, completion on an mbarrier) per work item.  Weights do not depend on
//                   activations, so the copies for the next phases are already in flight (or landed) while the consumers
//                   still wait at a grid barrier, stage an activation vector or run attention, until the ring is full
//                   (one ring is about 8 us of HBM time on an H100; DESIGN.md §5.2 has what the boundaries cost).
//   work item       (16-row tile, chunk of 2-5 consecutive 256-weight blocks): 16 x {110,144,176,210} bytes per block, contiguous
//                   in the STREAM layout written at load time (k_repack_stream).  Items are numbered in one sequence that both
//                   sides enumerate identically; item n belongs to consumer warp n % ST_W and lives in one of that warp's slots.
//   consumer warp   per block: the 8 (sub-block) x 8 (AVX lane) 4-element integer dots of 16 rows come from 8 tensor-core
//                   instructions — mma.sync.m16n8k32 u8 x s8 with A = 16 rows x one 32-weight sub-block (nibbles unpacked in
//                   registers) and B = that sub-block's int8 activations laid out BLOCK-DIAGONALLY (column l holds elements
//                   4l..4l+3, zero elsewhere), so D[row][l] is exactly what int32 lane l of the reference's AVX2 kernel holds
//                   after maddubs/madd.  Scales are folded with dp2a, the per-block fp32 terms (exact integers) are parked in
//                   registers, and the reference's fmadd chain per AVX lane is replayed IN BLOCK ORDER: a chunk that is not
//                   the first of its tile receives the running fp32 state of the 16 rows from the warp that folded the
//                   previous chunk (shared-memory mailbox + flag), folds its blocks and passes the state on; the last chunk
//                   ends with hsum_float_8's tree and the epilogue.  Any partition of a row therefore gives the same bits.
//   grid barrier    one atomic arrive + acquire spin per phase boundary (all phases depend on the whole previous output).
//
// Algorithmic HBM bytes: the GGUF bytes of the weights, once per token (same byte count in the stream layout).
#pragma once
#include <stdexcept>
#include <string>
#include "matvec.cuh"

namespace ctb {

#ifndef CTB_ST_WARPS
#define CTB_ST_WARPS 10
#endif
constexpr int ST_W = CTB_ST_WARPS;      // consumer warps
constexpr int ST_NT = ST_W * 32;        // consumer threads (threads 0 .. ST_NT-1)
constexpr int ST_THREADS = ST_NT + 32;  // + the producer warp
constexpr int ST_SLOT = 9216;           // ring slot: holds 5 Q3_K / 4 Q4_K / 3 Q5_K / 2 Q6_K blocks of a 16-row tile
#ifndef CTB_ST_DEPTH
#define CTB_ST_DEPTH 2
#endif
constexpr int ST_MAX_DEPTH = CTB_ST_DEPTH;   // slots per consumer warp; the ring has ST_W * depth slots
constexpr int ST_MAX_SLOTS = ST_W * ST_MAX_DEPTH;
constexpr int ST_MAXT = 16;             // tiles of a CTA whose fold chains are alive at the same time (one mailbox each)
constexpr int ST_ROWS = 16;
constexpr int ST_BAR = 1;               // named barrier of the consumer warps
constexpr int ST_STATE = 6;             // floats of fold state per thread: 4 AVX-lane accumulators + up to 2 mins accumulators

#ifndef CTB_CHUNK_Q3
#define CTB_CHUNK_Q3 5
#endif
#ifndef CTB_CHUNK_Q4
#define CTB_CHUNK_Q4 4
#endif
#ifndef CTB_CHUNK_Q5
#define CTB_CHUNK_Q5 3
#endif
#ifndef CTB_CHUNK_Q6
#define CTB_CHUNK_Q6 2
#endif
// Per K-quant type: bytes of one row's 256-weight block, blocks per work item (one ring slot), mins accumulators of the fold.
// Q3 = false: the kernels of programs without Q3_K matrices, whose arithmetic then has no trace of it (see k_step).
struct StType { int rb, kb, nm; };
template <bool Q3 = true>
__host__ __device__ constexpr StType st_type(int type) {
  return Q3 && type == GT_Q3_K ? StType{110, CTB_CHUNK_Q3, 0}
                               : (type == GT_Q4_K ? StType{144, CTB_CHUNK_Q4, 2} : (type == GT_Q5_K ? StType{176, CTB_CHUNK_Q5, 1} : StType{210, CTB_CHUNK_Q6, 0}));
}
template <int TYPE> struct StTraits {
  static constexpr int KB = st_type(TYPE).kb, BB = ST_ROWS * st_type(TYPE).rb, NM = st_type(TYPE).nm;
  static_assert(KB * BB <= ST_SLOT, "a work item must fit one ring slot");
};
__host__ __device__ inline int st_row_block_bytes(int type) { return st_type(type).rb; }
template <bool Q3 = true>
__host__ __device__ inline int st_block_bytes(int type) { return ST_ROWS * st_type<Q3>(type).rb; }   // 1760 / 2304 / 2816 / 3360
template <bool Q3 = true>
__host__ __device__ inline int st_chunk_blocks(int type) { return st_type<Q3>(type).kb; }
template <bool Q3 = true>
__host__ __device__ inline int st_tile_cost(int type) { return st_type<Q3>(type).rb / 2; }
// work items of a row of nb blocks (constant divisors)
template <bool Q3 = true>
__host__ __device__ inline int st_chunks(int type, int nb) {
  constexpr int K3 = StTraits<GT_Q3_K>::KB, K4 = StTraits<GT_Q4_K>::KB, K5 = StTraits<GT_Q5_K>::KB, K6 = StTraits<GT_Q6_K>::KB;
  if (Q3 && type == GT_Q3_K) return (nb + K3 - 1) / K3;
  return type == GT_Q4_K ? (nb + K4 - 1) / K4 : (type == GT_Q5_K ? (nb + K5 - 1) / K5 : (nb + K6 - 1) / K6);
}
__host__ __device__ inline size_t st_matrix_bytes(int type, int M, int nb) { return (size_t)((M + ST_ROWS - 1) / ST_ROWS) * nb * st_block_bytes(type); }

// ---------------------------------------------------------------------------------------------
// STREAM layout.  Tile i = rows 16i..16i+15; piece (i, b) = block b of those rows at byte ((i * nb + b) * st_block_bytes).
// Inside a piece, for mma thread (g = lane >> 2, t = lane & 3), h in {0,1} (AVX lane l = t + 4h), rr in {0,1} (row g + 8rr):
//   Q4_K  [0,2048)    16 B at ((h*2+rr)*32 + lane)*16: words j = 0..3 (32-weight pairs) of AVX lane l of that row  (k_quants.h:76-82)
//         [2048,2304) 16 B at (rr*8+g)*16: d, dmin, scales[12]
//   Q5_K  [0,2048)    as Q4_K;  [2048,2560) 4 B at ((h*2+rr)*32 + lane)*4: qh word l;  [2560,2816) headers      (k_quants.h:98-104)
//   Q6_K  [0,2048)    16 B: ql words (half 0, v 0) (0,1) (1,0) (1,1) of AVX lane l;  [2048,3072) 8 B at ((h*2+rr)*32 + lane)*8: qh
//         words of halves 0, 1;  [3072,3328) 16 int8 scales per row;  [3328,3360) fp16 d per row                (k_quants.h:112-117)
//   Q3_K  [0,1024)    8 B at ((h*2+rr)*32 + lane)*8: qs words of halves 0, 1 of AVX lane l;  [1024,1536) 4 B at ((h*2+rr)*32 +
//         lane)*4: hmask word l;  [1536,1728) the 12 scale bytes per row;  [1728,1760) fp16 d per row         (k_quants.h:55-61)
// A warp-wide 16-byte load of one (h, rr) plane touches 512 consecutive bytes: conflict-free.  Rows >= M are zero blocks.
__device__ __forceinline__ void st_decode(int type, int o, int& rl, int& src) {
  if (type == GT_Q3_K) {   // raw block: hmask[32] qs[64] scales[12] d
    if (o < 1536) {
      const bool qs = o < 1024;
      const int r = qs ? o : o - 1024, q = qs ? r >> 3 : r >> 2, hr = q >> 5, lane = q & 31, h = hr >> 1, rr = hr & 1, g = lane >> 2, t = lane & 3;
      rl = rr * 8 + g;
      src = (qs ? 32 + ((r >> 2) & 1) * 32 : 0) + 4 * (t + 4 * h) + (r & 3);
      return;
    }
    if (o < 1728) { const int r = o - 1536; rl = r / 12; src = 96 + r % 12; return; }
    rl = (o - 1728) >> 1; src = 108; return;
  }
  const int q4 = (type == GT_Q6_K) ? 0 : (type == GT_Q5_K ? 48 : 16);   // raw offset of the 128 nibble bytes
  if (o < 2048) {
    const int q = o >> 4, hr = q >> 5, lane = q & 31, h = hr >> 1, rr = hr & 1, g = lane >> 2, t = lane & 3, l = t + 4 * h;
    const int wi = (o >> 2) & 3, byte = o & 3;
    rl = rr * 8 + g;
    src = type == GT_Q6_K ? ((wi >> 1) * 64 + (wi & 1) * 32 + 4 * l + byte) : (q4 + 32 * wi + 4 * l + byte);
    return;
  }
  if (type == GT_Q4_K) { const int r = o - 2048; rl = r >> 4; src = r & 15; return; }
  if (type == GT_Q5_K) {
    if (o < 2560) {
      const int q = (o - 2048) >> 2, hr = q >> 5, lane = q & 31, h = hr >> 1, rr = hr & 1, g = lane >> 2, t = lane & 3;
      rl = rr * 8 + g; src = 16 + 4 * (t + 4 * h) + (o & 3);
      return;
    }
    const int r = o - 2560; rl = r >> 4; src = r & 15; return;
  }
  if (o < 3072) {
    const int r = o - 2048, q = r >> 3, hr = q >> 5, lane = q & 31, h = hr >> 1, rr = hr & 1, g = lane >> 2, t = lane & 3;
    rl = rr * 8 + g; src = 128 + ((r >> 2) & 1) * 32 + 4 * (t + 4 * h) + (r & 3);
    return;
  }
  if (o < 3328) { const int r = o - 3072; rl = r >> 4; src = 192 + (r & 15); return; }
  rl = (o - 3328) >> 1; src = 208;
}

// GGUF array-of-blocks → stream layout, 2 bytes per thread-iteration
static __global__ void k_repack_stream(int type, const uint8_t* __restrict__ raw, int M, int nb, uint16_t* __restrict__ st) {
  const int rbb = st_row_block_bytes(type), half = rbb * ST_ROWS / 2;
  const size_t n_units = (size_t)((M + ST_ROWS - 1) / ST_ROWS) * nb * half;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n_units; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t piece = idx / half;
    const int o = (int)(idx % half) * 2;
    const size_t tile = piece / nb;
    const int b = (int)(piece % nb);
    int rl, src;
    st_decode(type, o, rl, src);
    const size_t row = tile * ST_ROWS + rl;
    st[idx] = row < (size_t)M ? *(const uint16_t*)(raw + (row * nb + b) * rbb + src) : (uint16_t)0;
  }
}

// ---------------------------------------------------------------------------------------------
// Ring addressing.  Every owner (a consumer warp here, a team of warps in prefill.cuh) has its own `depth` slots: its i-th
// item lives in slot (i % depth) * owners + owner with mbarrier phase parity (i / depth) & 1.  The owner that waits for an item
// is the one that consumed the slot's previous occupant, so it can never be a whole barrier phase ahead of the data (a parity
// wait cannot tell phase r from phase r + 2: with slots shared between owners a fast warp saw "full" on a slot whose previous
// item was still landing).
struct RingPos { uint32_t slot, parity; };
__device__ __forceinline__ RingPos ring_pos(uint32_t i, uint32_t owner, uint32_t owners, uint32_t depth) { return {(i % depth) * owners + owner, (i / depth) & 1u}; }
// the step kernel's items form one sequence that the producer and the consumers enumerate identically; item n belongs to warp n % ST_W
__device__ __forceinline__ RingPos st_ring(uint32_t n, uint32_t depth) { return ring_pos(n / ST_W, n % ST_W, ST_W, depth); }

// ---------------------------------------------------------------------------------------------
// PTX: mbarrier, bulk copy, tensor-core mma
__device__ __forceinline__ uint32_t st_smem(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(st_smem(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(st_smem(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(st_smem(bar)) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(st_smem(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, WaitCode code, int aux) {
  bounded_wait([&] { return mbar_try_wait(bar, parity); }, code, aux);
}
// the ring's barriers, by thread 0 before the CTA's first barrier: a full barrier completes on the producer's arrive and the
// bytes of its copy, an empty barrier on the arrives of the consumers that share a slot
__device__ __forceinline__ void ring_init(uint64_t* full_bar, uint64_t* empty_bar, int n_slots, int consumers_per_slot) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < n_slots; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], consumers_per_slot); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
}
// global → shared bulk copy (TMA, SASS UBLKCP), completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(st_smem(dst)), "l"(src), "r"(bytes), "r"(st_smem(bar)) : "memory");
}
// the same with an L2 cache policy (createpolicy) for the lines it reads
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(st_smem(dst)), "l"(src), "r"(bytes),
               "r"(st_smem(bar)), "l"(pol) : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// D(16x8, s32) = A(16x32, u8, row) · B(32x8, s8, col) + C.  Fragments (PTX ISA, m16n8k32 8-bit): a0 = row g, k 4t..4t+3; a1 = row
// g+8, same k; a2 = row g, k 16+4t..; a3 = row g+8, k 16+4t..;  b0 = k 4t..4t+3, col g;  b1 = k 16+4t.., col g;  d0/d1 = row g,
// cols 2t, 2t+1;  d2/d3 = row g+8, cols 2t, 2t+1.
__device__ __forceinline__ void mma_u8s8(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1, int c0, int c1) {
  asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
      : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(c0), "r"(c1), "r"(c0), "r"(c1));
}

// ---------------------------------------------------------------------------------------------
// Activation vector in shared memory: the Q8_K image written by stage_activation (qs lane-major per block, d, bsums) plus
//   pairs  per block 4 words: (bsums[4k]+bsums[4k+1]) | (bsums[4k+2]+bsums[4k+3]) << 16 — the operands of the Q4_K / Q5_K mins terms
//   cneg   Q6_K / Q3_K phases: per block [t][group][c] int32 = -32 · Σ of the 4 activations of AVX lane l = 2t+c of 32-weight group
//          `group`: the accumulator input that turns u·q8 into (u-32)·q8 (the AVX2 kernel subtracts maddubs(32, q8), k_quants.c:3829-3843);
//          Q3_K takes cneg / 8, which turns u·q8 into (u-4)·q8
struct StAct {
  const int8_t* qs;
  const float* d;
  const uint32_t* pairs;
  const int* cneg;
  const int8_t* zero;   // 256 zero bytes (what the off-diagonal lanes of the mma B operand read)
  const struct XchgParams* xc;   // non-null: the phase produces a tensor-parallel exchange (rows go to every rank's ll slots)
  unsigned epoch;
};
__host__ __device__ inline size_t st_off_pairs(int K) { return ((((size_t)K + 15) & ~(size_t)15) + q8k_d_bytes(K) + (size_t)(K / 16) * 2 + 15) & ~(size_t)15; }
__host__ __device__ inline size_t st_act_bytes(int K, bool q6) { return st_off_pairs(K) + (size_t)(K / 256) * 16 + (q6 ? (size_t)K : 0) + 256 + 16; }

template <int NT, int BAR>
__device__ __forceinline__ StAct st_act_extras(uint8_t* smem, int K, bool q6) {
  const ActView a = act_view(ACT_Q8_K, K, smem);
  StAct s;
  s.qs = a.qs; s.d = a.d;
  uint32_t* pairs = (uint32_t*)(smem + st_off_pairs(K));
  int* cneg = (int*)(smem + st_off_pairs(K) + (size_t)(K / 256) * 16);
  s.pairs = pairs; s.cneg = cneg;
  const int nb = K >> 8;
  int* zero = (int*)(smem + st_off_pairs(K) + (size_t)nb * 16 + (q6 ? (size_t)K : 0));
  s.zero = (const int8_t*)zero;
  if (threadIdx.x < 64) zero[threadIdx.x] = 0;
  for (int i = threadIdx.x; i < nb * 4; i += NT) {
    const int16_t* b4 = a.bs + (i >> 2) * 16 + 4 * (i & 3);
    const int p0 = (int)b4[0] + (int)b4[1], p1 = (int)b4[2] + (int)b4[3];
    pairs[i] = (uint32_t)(p0 & 0xffff) | ((uint32_t)p1 << 16);
  }
  if (q6) {
    for (int i = threadIdx.x; i < nb * 64; i += NT) {
      const int b = i >> 6, grp = (i >> 3) & 7, l = i & 7;
      const int w = *(const int*)(a.qs + q8k_word_offset(b, grp, l));
      cneg[((b * 4 + (l >> 1)) * 8 + grp) * 2 + (l & 1)] = -32 * __dp4a(0x01010101, w, 0);
    }
  }
  bar_sync<BAR, NT>();
  return s;
}

// unpack the 12 scale bytes of a Q4_K/Q5_K header (k_quants.c:306-313 get_scale_min_k4, all 8 at once)
__device__ __forceinline__ void unpack_k4(uint32_t s0, uint32_t s1, uint32_t s2, uint32_t& sc03, uint32_t& sc47, uint32_t& m03, uint32_t& m47) {
  sc03 = s0 & 0x3f3f3f3fu;
  m03 = s1 & 0x3f3f3f3fu;
  sc47 = (s2 & 0x0f0f0f0fu) | (((s0 >> 6) & 0x03030303u) << 4);
  m47 = ((s2 >> 4) & 0x0f0f0f0fu) | (((s1 >> 6) & 0x03030303u) << 4);
}
__device__ __forceinline__ int pack16(int lo, int hi) { return (int)__byte_perm((uint32_t)lo, (uint32_t)hi, 0x5410); }
// Σ_s scale_s · dot_s over the 8 sub-block dots of one (row, AVX lane); every dot fits int16, the scales are bytes
__device__ __forceinline__ int scale_fold8(int d0, int d1, int d2, int d3, int d4, int d5, int d6, int d7, uint32_t s03, uint32_t s47) {
  int s = __dp2a_lo(pack16(d0, d1), (int)s03, 0);
  s = __dp2a_hi(pack16(d2, d3), (int)s03, s);
  s = __dp2a_lo(pack16(d4, d5), (int)s47, s);
  s = __dp2a_hi(pack16(d6, d7), (int)s47, s);
  return s;
}

// What one block contributes to this thread's share of the 16 rows: p[rr*2+c] = (float) of int32 lane l = 2t+c of row g+8rr;
// dd[rr] = y.d·d; mins: Q4_K pm[rr] = mins lane k = t of row g+8rr (ddm[rr] = -y.d·dmin); Q5_K pm[0] = the scalar mins term of
// row g+8(t&1) (ddm[0]); Q3_K / Q6_K none.
struct Terms { float p[4]; float pm[2]; float dd[2]; float ddm[2]; };

__device__ __forceinline__ void load_b_operands(const StAct& a, int b, int g, int t, uint32_t (&bA)[8], uint32_t (&bB)[8]) {
  // block-diagonal B: thread (g, t) holds rows 4t..4t+3 / 16+4t.. of column g, which are non-zero only for g == t / g == t+4.
  // Branch-free (ptxas interleaves the blocks of an item): the off-diagonal lanes load from a run of zero bytes instead.
  const int8_t* word = a.qs + b * 256 + g * 16;
  const int8_t* pa = (g == t) ? word : a.zero;
  const int8_t* pb = (g == t + 4) ? word : a.zero;
  const int4 la = *(const int4*)pa, ha = *(const int4*)(pa + 128), lb = *(const int4*)pb, hb = *(const int4*)(pb + 128);
  bA[0] = la.x; bA[1] = la.y; bA[2] = la.z; bA[3] = la.w; bA[4] = ha.x; bA[5] = ha.y; bA[6] = ha.z; bA[7] = ha.w;
  bB[0] = lb.x; bB[1] = lb.y; bB[2] = lb.z; bB[3] = lb.w; bB[4] = hb.x; bB[5] = hb.y; bB[6] = hb.z; bB[7] = hb.w;
}

template <int TYPE>
__device__ __forceinline__ void block_terms(const uint8_t* blk, int b, const StAct& a, int lane, Terms& r);

// k_quants.c:2651-2714
template <>
__device__ __forceinline__ void block_terms<GT_Q4_K>(const uint8_t* blk, int b, const StAct& a, int lane, Terms& r) {
  const int g = lane >> 2, t = lane & 3;
  const int4* qp = (const int4*)blk;
  const int4 w00 = qp[lane], w01 = qp[32 + lane], w10 = qp[64 + lane], w11 = qp[96 + lane];
  const int4 h0 = ((const int4*)(blk + 2048))[g], h1 = ((const int4*)(blk + 2048))[8 + g];
  uint32_t bA[8], bB[8];
  load_b_operands(a, b, g, t, bA, bB);
  const uint32_t W[4][4] = {{(uint32_t)w00.x, (uint32_t)w01.x, (uint32_t)w10.x, (uint32_t)w11.x}, {(uint32_t)w00.y, (uint32_t)w01.y, (uint32_t)w10.y, (uint32_t)w11.y},
                            {(uint32_t)w00.z, (uint32_t)w01.z, (uint32_t)w10.z, (uint32_t)w11.z}, {(uint32_t)w00.w, (uint32_t)w01.w, (uint32_t)w10.w, (uint32_t)w11.w}};
  int D[8][4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    mma_u8s8(D[2 * j], W[j][0] & 0x0f0f0f0fu, W[j][1] & 0x0f0f0f0fu, W[j][2] & 0x0f0f0f0fu, W[j][3] & 0x0f0f0f0fu, bA[2 * j], bB[2 * j], 0, 0);
    mma_u8s8(D[2 * j + 1], (W[j][0] >> 4) & 0x0f0f0f0fu, (W[j][1] >> 4) & 0x0f0f0f0fu, (W[j][2] >> 4) & 0x0f0f0f0fu, (W[j][3] >> 4) & 0x0f0f0f0fu, bA[2 * j + 1],
             bB[2 * j + 1], 0, 0);
  }
  const float yd = a.d[b];
  const uint32_t pw = a.pairs[b * 4 + t];
#pragma unroll
  for (int rr = 0; rr < 2; rr++) {
    const int4 h = rr ? h1 : h0;
    uint32_t sc03, sc47, m03, m47;
    unpack_k4((uint32_t)h.y, (uint32_t)h.z, (uint32_t)h.w, sc03, sc47, m03, m47);
#pragma unroll
    for (int c = 0; c < 2; c++) {
      const int i = rr * 2 + c;
      r.p[i] = (float)scale_fold8(D[0][i], D[1][i], D[2][i], D[3][i], D[4][i], D[5][i], D[6][i], D[7][i], sc03, sc47);
    }
    r.dd[rr] = __fmul_rn(yd, h2f((uint16_t)((uint32_t)h.x & 0xffffu)));
    r.ddm[rr] = __fmul_rn(-yd, h2f((uint16_t)((uint32_t)h.x >> 16)));
    // mins lane k = t: m[2k]·(bsums[4k]+bsums[4k+1]) + m[2k+1]·(bsums[4k+2]+bsums[4k+3])
    const uint32_t mw = (t < 2 ? m03 : m47) >> ((t & 1) * 16);
    r.pm[rr] = (float)__dp2a_lo((int)pw, (int)mw, 0);
  }
}

// k_quants.c:3174-3262
template <>
__device__ __forceinline__ void block_terms<GT_Q5_K>(const uint8_t* blk, int b, const StAct& a, int lane, Terms& r) {
  const int g = lane >> 2, t = lane & 3;
  const int4* qp = (const int4*)blk;
  const int4 w00 = qp[lane], w01 = qp[32 + lane], w10 = qp[64 + lane], w11 = qp[96 + lane];
  const uint32_t* hp = (const uint32_t*)(blk + 2048);
  const uint32_t HB[4] = {hp[lane], hp[32 + lane], hp[64 + lane], hp[96 + lane]};
  const int4 h0 = ((const int4*)(blk + 2560))[g], h1 = ((const int4*)(blk + 2560))[8 + g];
  uint32_t bA[8], bB[8];
  load_b_operands(a, b, g, t, bA, bB);
  const uint32_t W[4][4] = {{(uint32_t)w00.x, (uint32_t)w01.x, (uint32_t)w10.x, (uint32_t)w11.x}, {(uint32_t)w00.y, (uint32_t)w01.y, (uint32_t)w10.y, (uint32_t)w11.y},
                            {(uint32_t)w00.z, (uint32_t)w01.z, (uint32_t)w10.z, (uint32_t)w11.z}, {(uint32_t)w00.w, (uint32_t)w01.w, (uint32_t)w10.w, (uint32_t)w11.w}};
  int D[8][4];
#pragma unroll
  for (int j = 0; j < 4; j++) {   // bit s of a qh byte: 5th bit of the element in sub-block s
    uint32_t lo[4], hi[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      lo[i] = (W[j][i] & 0x0f0f0f0fu) | (((HB[i] >> (2 * j)) & 0x01010101u) << 4);
      hi[i] = ((W[j][i] >> 4) & 0x0f0f0f0fu) | (((HB[i] >> (2 * j + 1)) & 0x01010101u) << 4);
    }
    mma_u8s8(D[2 * j], lo[0], lo[1], lo[2], lo[3], bA[2 * j], bB[2 * j], 0, 0);
    mma_u8s8(D[2 * j + 1], hi[0], hi[1], hi[2], hi[3], bA[2 * j + 1], bB[2 * j + 1], 0, 0);
  }
  const float yd = a.d[b];
  const uint4 pw = *(const uint4*)(a.pairs + b * 4);
#pragma unroll
  for (int rr = 0; rr < 2; rr++) {
    const int4 h = rr ? h1 : h0;
    uint32_t sc03, sc47, m03, m47;
    unpack_k4((uint32_t)h.y, (uint32_t)h.z, (uint32_t)h.w, sc03, sc47, m03, m47);
#pragma unroll
    for (int c = 0; c < 2; c++) {
      const int i = rr * 2 + c;
      r.p[i] = (float)scale_fold8(D[0][i], D[1][i], D[2][i], D[3][i], D[4][i], D[5][i], D[6][i], D[7][i], sc03, sc47);
    }
    r.dd[rr] = __fmul_rn(yd, h2f((uint16_t)((uint32_t)h.x & 0xffffu)));
    {   // the scalar mins term of the AVX2 kernel: Σ_k m[k]·(bsums[2k]+bsums[2k+1]), kept by thread t = rr of the row's quad
      int hs = __dp2a_lo((int)pw.x, (int)m03, 0);
      hs = __dp2a_hi((int)pw.y, (int)m03, hs);
      hs = __dp2a_lo((int)pw.z, (int)m47, hs);
      hs = __dp2a_hi((int)pw.w, (int)m47, hs);
      const float pmv = (float)hs, dmv = __fmul_rn(-yd, h2f((uint16_t)((uint32_t)h.x >> 16)));
      if (rr == 0) { r.pm[0] = pmv; r.ddm[0] = dmv; }
      else { r.pm[0] = (t & 1) ? pmv : r.pm[0]; r.ddm[0] = (t & 1) ? dmv : r.ddm[0]; }
    }
  }
}

// k_quants.c:3794-3872
template <>
__device__ __forceinline__ void block_terms<GT_Q6_K>(const uint8_t* blk, int b, const StAct& a, int lane, Terms& r) {
  const int g = lane >> 2, t = lane & 3;
  const int4* qp = (const int4*)blk;
  const int2* hp = (const int2*)(blk + 2048);
  const int4 QL[4] = {qp[lane], qp[32 + lane], qp[64 + lane], qp[96 + lane]};   // index h*2+rr; words (half 0: A, B) (half 1: A, B)
  const int2 QH[4] = {hp[lane], hp[32 + lane], hp[64 + lane], hp[96 + lane]};
  const int4 s0 = ((const int4*)(blk + 3072))[g], s1 = ((const int4*)(blk + 3072))[8 + g];
  const uint16_t d0 = ((const uint16_t*)(blk + 3328))[g], d1 = ((const uint16_t*)(blk + 3328))[8 + g];
  uint32_t bA[8], bB[8];
  load_b_operands(a, b, g, t, bA, bB);
  const int4* cp = (const int4*)(a.cneg + (b * 4 + t) * 16);   // [group][c] for this thread's two columns
  const int4 cn[4] = {cp[0], cp[1], cp[2], cp[3]};
  const int C[8][2] = {{cn[0].x, cn[0].y}, {cn[0].z, cn[0].w}, {cn[1].x, cn[1].y}, {cn[1].z, cn[1].w}, {cn[2].x, cn[2].y}, {cn[2].z, cn[2].w}, {cn[3].x, cn[3].y}, {cn[3].z, cn[3].w}};
  int D[8][4];
#pragma unroll
  for (int jj = 0; jj < 2; jj++) {
    uint32_t u[4][4];   // [m][fragment register]
#pragma unroll
    for (int i = 0; i < 4; i++) {
      // fragment register order a0..a3 = (h0,rr0) (h0,rr1) (h1,rr0) (h1,rr1) = plane index i
      const uint32_t A = (uint32_t)(jj ? QL[i].z : QL[i].x), B = (uint32_t)(jj ? QL[i].w : QL[i].y), H = (uint32_t)(jj ? QH[i].y : QH[i].x);
      u[0][i] = (A & 0x0f0f0f0fu) | ((H << 4) & 0x30303030u);
      u[1][i] = (B & 0x0f0f0f0fu) | ((H << 2) & 0x30303030u);
      u[2][i] = ((A >> 4) & 0x0f0f0f0fu) | (H & 0x30303030u);
      u[3][i] = ((B >> 4) & 0x0f0f0f0fu) | ((H >> 2) & 0x30303030u);
    }
#pragma unroll
    for (int m = 0; m < 4; m++) {
      const int grp = jj * 4 + m;
      mma_u8s8(D[grp], u[m][0], u[m][1], u[m][2], u[m][3], bA[grp], bB[grp], C[grp][0], C[grp][1]);
    }
  }
  const float yd = a.d[b];
  const int par = t >> 1;   // this thread's columns 2t, 2t+1 are AVX lanes of the first (par 0) or second (par 1) 16 weights of each group
#pragma unroll
  for (int rr = 0; rr < 2; rr++) {
    const int4 sv = rr ? s1 : s0;
    // int8 scale of (half jj, group m, par): byte 2(m&1)+par of word jj*2+(m>>1) -> S[jj] = scales of m = 0..3 as 4 signed bytes
    const uint32_t sel = par ? 0x7531u : 0x6420u;
    const uint32_t S0 = __byte_perm((uint32_t)sv.x, (uint32_t)sv.y, sel), S1 = __byte_perm((uint32_t)sv.z, (uint32_t)sv.w, sel);
#pragma unroll
    for (int c = 0; c < 2; c++) {
      const int i = rr * 2 + c;
      r.p[i] = (float)scale_fold8(D[0][i], D[1][i], D[2][i], D[3][i], D[4][i], D[5][i], D[6][i], D[7][i], S0, S1);
    }
    r.dd[rr] = __fmul_rn(yd, h2f(rr ? d1 : d0));
  }
}

// k_quants.c:1950-2052.  The weight u = q3l | (hbit << 2) in [0, 7] is the u8 operand; the reference's value is u - 4, and the
// -4 rides in as the accumulator input: -4 · Σ of the lane's 4 activations = cneg / 8 (exact: cneg is a multiple of 32).  Every
// D fits int16 (|u - 4| <= 4, 4 products of |q8| <= 128), as scale_fold8 needs.
template <>
__device__ __forceinline__ void block_terms<GT_Q3_K>(const uint8_t* blk, int b, const StAct& a, int lane, Terms& r) {
  const int g = lane >> 2, t = lane & 3;
  const int2* qp = (const int2*)blk;
  const uint32_t* hp = (const uint32_t*)(blk + 1024);
  const int2 QS[4] = {qp[lane], qp[32 + lane], qp[64 + lane], qp[96 + lane]};   // index h*2+rr; words of halves 0, 1
  const uint32_t HM[4] = {hp[lane], hp[32 + lane], hp[64 + lane], hp[96 + lane]};
  const uint32_t* sp = (const uint32_t*)(blk + 1536);
  const uint32_t sa[2][3] = {{sp[3 * g], sp[3 * g + 1], sp[3 * g + 2]}, {sp[3 * (8 + g)], sp[3 * (8 + g) + 1], sp[3 * (8 + g) + 2]}};
  const uint16_t d0 = ((const uint16_t*)(blk + 1728))[g], d1 = ((const uint16_t*)(blk + 1728))[8 + g];
  uint32_t bA[8], bB[8];
  load_b_operands(a, b, g, t, bA, bB);
  const int4* cp = (const int4*)(a.cneg + (b * 4 + t) * 16);   // [group][c] for this thread's two columns
  const int4 cn[4] = {cp[0], cp[1], cp[2], cp[3]};
  const int C[8][2] = {{cn[0].x, cn[0].y}, {cn[0].z, cn[0].w}, {cn[1].x, cn[1].y}, {cn[1].z, cn[1].w}, {cn[2].x, cn[2].y}, {cn[2].z, cn[2].w}, {cn[3].x, cn[3].y}, {cn[3].z, cn[3].w}};
  int D[8][4];
#pragma unroll
  for (int grp = 0; grp < 8; grp++) {   // 32-weight group grp = 4j + k: bits 2k of qs word j, bit grp of the hmask byte
    uint32_t u[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t q = (uint32_t)(grp < 4 ? QS[i].x : QS[i].y);
      u[i] = ((q >> (2 * (grp & 3))) & 0x03030303u) | (((HM[i] >> grp) & 0x01010101u) << 2);
    }
    mma_u8s8(D[grp], u[0], u[1], u[2], u[3], bA[grp], bB[grp], C[grp][0] >> 3, C[grp][1] >> 3);
  }
  const float yd = a.d[b];
  const int par = t >> 1;   // this thread's columns 2t, 2t+1 are AVX lanes of the first (par 0) or second (par 1) 16 weights of each group
#pragma unroll
  for (int rr = 0; rr < 2; rr++) {
    // the 16 six-bit scales (k_quants.c:1968-1974), minus 32 per byte: word w holds sub-blocks 4w .. 4w+3
    const uint32_t a0 = sa[rr][0], a1 = sa[rr][1], a2 = sa[rr][2];
    const uint32_t w0 = __vsub4((a0 & 0x0f0f0f0fu) | ((a2 & 0x03030303u) << 4), 0x20202020u);
    const uint32_t w1 = __vsub4((a1 & 0x0f0f0f0fu) | (((a2 >> 2) & 0x03030303u) << 4), 0x20202020u);
    const uint32_t w2 = __vsub4(((a0 >> 4) & 0x0f0f0f0fu) | (((a2 >> 4) & 0x03030303u) << 4), 0x20202020u);
    const uint32_t w3 = __vsub4(((a1 >> 4) & 0x0f0f0f0fu) | (((a2 >> 6) & 0x03030303u) << 4), 0x20202020u);
    // scale of (group grp, par) = sub-block 2grp + par: S0 = groups 0..3, S1 = groups 4..7, as 4 signed bytes
    const uint32_t sel = par ? 0x7531u : 0x6420u;
    const uint32_t S0 = __byte_perm(w0, w1, sel), S1 = __byte_perm(w2, w3, sel);
#pragma unroll
    for (int c = 0; c < 2; c++) {
      const int i = rr * 2 + c;
      r.p[i] = (float)scale_fold8(D[0][i], D[1][i], D[2][i], D[3][i], D[4][i], D[5][i], D[6][i], D[7][i], S0, S1);
    }
    r.dd[rr] = __fmul_rn(yd, h2f(rr ? d1 : d0));
  }
}

// One work item: blocks [b0, b0 + nblk) of the 16-row tile whose pieces lie in `slot`.  Integer work first (the slot is
// released as soon as the last weight word has been read), then the ordered fp32 fold: state in from the mailbox unless this
// is the tile's first chunk, blocks folded in order, state out unless it is the last chunk — then hsum_float_8 and the epilogue.
template <int TYPE, bool XC>
__device__ __forceinline__ void run_item(const uint8_t* slot, uint64_t* empty_bar, int nblk, int b0, int kc, bool last, const StAct& a, int lane,
                                         volatile float* mail, volatile int* flag, const MVSeg& sg, const MVParams& p, int row0) {
  constexpr int KB = StTraits<TYPE>::KB, BB = StTraits<TYPE>::BB, NM = StTraits<TYPE>::NM;
  Terms tr[KB];
  if (nblk == KB) {   // the common case, straight-line: the KB blocks are independent until the fold, ptxas interleaves them
#pragma unroll
    for (int i = 0; i < KB; i++) block_terms<TYPE>(slot + i * BB, b0 + i, a, lane, tr[i]);
  } else {
#pragma unroll
    for (int i = 0; i < KB; i++) {
      if (i < nblk) block_terms<TYPE>(slot + i * BB, b0 + i, a, lane, tr[i]);
      else { Terms z{}; tr[i] = z; }
    }
  }
  __syncwarp();
  if (lane == 0) mbar_arrive(empty_bar);   // every lane has its weight words in registers: the producer may refill the slot

  float acc[4] = {0.f, 0.f, 0.f, 0.f}, accm[2] = {0.f, 0.f};
  if (kc > 0) {
    if (lane == 0) bounded_wait([&] { return *flag >= kc; }, W_FOLD_FLAG, kc);
    __syncwarp();
    __threadfence_block();
#pragma unroll
    for (int i = 0; i < 4; i++) acc[i] = mail[i * 32 + lane];
#pragma unroll
    for (int i = 0; i < NM; i++) accm[i] = mail[(4 + i) * 32 + lane];
  }
#pragma unroll
  for (int i = 0; i < KB; i++) {
    if (i < nblk) {   // (a skipped block must not touch the accumulators: fma(0, 0, -0.0f) would flip a sign bit)
      // one fmadd per block and AVX lane, blocks in order (k_quants.c:2048, 2706, 3253, 3864); mins: 2699-2701 (Q4_K), 3199-3201 (Q5_K)
#pragma unroll
      for (int q = 0; q < 4; q++) acc[q] = __fmaf_rn(tr[i].dd[q >> 1], tr[i].p[q], acc[q]);
#pragma unroll
      for (int q = 0; q < NM; q++) accm[q] = __fmaf_rn(tr[i].ddm[q], tr[i].pm[q], accm[q]);
    }
  }
  if (!last) {
    __syncwarp();   // all lanes have read the incoming state before anybody overwrites the mailbox
#pragma unroll
    for (int i = 0; i < 4; i++) mail[i * 32 + lane] = acc[i];
#pragma unroll
    for (int i = 0; i < NM; i++) mail[(4 + i) * 32 + lane] = accm[i];
    __threadfence_block();
    __syncwarp();
    if (lane == 0) *flag = kc + 1;
    return;
  }
  // hsum_float_8 (ggml.c:609-615): res[l] = x[l] + x[l+4]; (res[0]+res[2]) + (res[1]+res[3]).  Thread t holds x[2t], x[2t+1].
  const int t = lane & 3, g = lane >> 2;
  float out[2];
#pragma unroll
  for (int rr = 0; rr < 2; rr++) {
    float u0 = acc[rr * 2], u1 = acc[rr * 2 + 1];
    u0 = __fadd_rn(u0, __shfl_xor_sync(0xffffffffu, u0, 2));   // t = 0: x0+x4, t = 1: x2+x6
    u1 = __fadd_rn(u1, __shfl_xor_sync(0xffffffffu, u1, 2));   // t = 0: x1+x5, t = 1: x3+x7
    u0 = __fadd_rn(u0, __shfl_xor_sync(0xffffffffu, u0, 1));   // res[0]+res[2]
    u1 = __fadd_rn(u1, __shfl_xor_sync(0xffffffffu, u1, 1));   // res[1]+res[3]
    float v = __fadd_rn(u0, u1);
    if (TYPE == GT_Q4_K) {          // acc_m: (m0+m2) + (m1+m3), then added to the total (k_quants.c:2709-2712)
      float m = accm[rr];
      m = __fadd_rn(m, __shfl_xor_sync(0xffffffffu, m, 2));
      m = __fadd_rn(m, __shfl_xor_sync(0xffffffffu, m, 1));
      v = __fadd_rn(v, m);
    } else if (TYPE == GT_Q5_K) {   // the scalar mins chain of row g+8rr lives in thread t = rr of the quad
      v = __fadd_rn(v, __shfl_sync(0xffffffffu, accm[0], (lane & ~3) + rr));
    }
    out[rr] = v;
  }
  if (t < 2) {
    const int row = row0 + g + 8 * t;
    if (row < sg.w.M) {
      if (XC && a.xc) {   // tensor-parallel partial sum: {value (+ residual on the rank that carries it), exchange number} to every rank
        const float v = epilogue(sg.epi, t ? out[1] : out[0], sg.res + row, sg.res2 + row, p);
        const XchgParams& xc = *a.xc;
        const size_t at = ((size_t)(a.epoch & 1u) * xc.world + xc.rank) * xc.n + row;
        for (int r = 0; r < xc.world; r++)
          asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(xc.ll[r] + at), "r"(__float_as_uint(v)), "r"(a.epoch) : "memory");
      } else {
        store_epilogue(sg, p, row, t ? out[1] : out[0]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// The 16-row tiles of a phase's matrices, concatenated; CTA c owns a contiguous, byte-balanced range of them.
struct TileSpace {
  int tiles[MV_MAX_SEG], cost[MV_MAX_SEG], nseg, ntiles;
  long total;   // Σ tiles·cost
  template <bool Q3 = true>
  __host__ __device__ __forceinline__ void init(const MVParams& p) {
    nseg = p.nseg; ntiles = 0; total = 0;
#pragma unroll
    for (int s = 0; s < MV_MAX_SEG; s++) {
      tiles[s] = s < p.nseg ? (p.seg[s].w.M + ST_ROWS - 1) / ST_ROWS : 0;
      cost[s] = s < p.nseg ? st_tile_cost<Q3>(p.seg[s].w.type) : 1;
      ntiles += tiles[s]; total += (long)tiles[s] * cost[s];
    }
  }
  // matrix a tile of the concatenated space belongs to; `tile` becomes the tile index inside that matrix
  __host__ __device__ __forceinline__ int locate(int& tile) const {
    static_assert(MV_MAX_SEG == 3, "locate() is written out for three segments");
    if (tile < tiles[0]) return 0;
    tile -= tiles[0];
    if (tile < tiles[1]) return 1;
    tile -= tiles[1];
    return 2;
  }
  // first tile of CTA c of G: the tile at which the cumulative cost reaches c/G of the total
  __host__ __device__ __forceinline__ int boundary(int c, int G) const {
    if (c >= G) return ntiles;
    long target = total * c / G;
    int base = 0;
#pragma unroll
    for (int s = 0; s < MV_MAX_SEG; s++) {
      const long span = (long)tiles[s] * cost[s];
      if (target < span || s == MV_MAX_SEG - 1) return base + (int)min((long)tiles[s], (target + cost[s] / 2) / cost[s]);
      target -= span; base += tiles[s];
    }
    return ntiles;
  }
};

// ---------------------------------------------------------------------------------------------
// Phases of a step
enum : int { PH_MATVEC = 0, PH_ATTN = 1, PH_EMBED = 2, PH_PICK = 3,
              PH_XCHG = 4 };   // PH_XCHG: host-side schedule entry only (tensor-parallel NCCL all-reduce between two launches), never a kernel phase
// Tensor-parallel exchange fused into the step (peer memory over NVLink; no kernel boundary, no NCCL call, no fence).  Every rank
// owns a region  uint2 ll[2][world][n]  that all ranks have mapped (CUDA IPC); an element is {float bits, exchange number} and is
// always written with ONE 8-byte store, so a reader that sees the right exchange number sees the value that came with it (the
// "LL" idea of NCCL's low-latency protocol).  The row-parallel phase (role 2) stores every finished output row of this rank,
// residual included on rank 0, into ll[parity][rank][row] of EVERY rank straight from its epilogue; the next mat-vec phase
// (role 1) stages  x = ll[parity][0] + ll[parity][1] + ...  (rank order: every rank forms the same bits), spinning on elements
// whose number is not there yet.  The copies ride under the local grid barrier, so an exchange costs about one NVLink hop.
// Two parities suffice: a rank can produce exchange k+2 only after it has consumed k+1, which its peers produce after they
// have finished reading k.
constexpr int XC_MAX_WORLD = 8;
struct XchgParams {
  int world, rank, index, n;           // index: number of this exchange inside the program (0-based); n: elements per vector
  int role;                            // 0 none, 1 this phase consumes the exchange (sums it while staging), 2 it produces it
  uint2* ll[XC_MAX_WORLD];             // region base of every rank as mapped here
};
// The number an element of exchange `index` (0-based inside the program) carries in a launch that starts after `base` exchanges
// (StepArgs::sync[2]); its parity half of the regions is the number's low bit.  The numbers wrap past 2^32 without a break.
__host__ __device__ inline unsigned xc_epoch(unsigned base, int index) { return base + (unsigned)index + 1u; }
struct PickParams { const float* logits; int* state; int* out_tokens; int n; };
struct alignas(16) Phase {
  int kind;
  int q6;           // PH_MATVEC: some matrix of the phase is Q6_K or Q3_K (the activation staging then also builds cneg)
                    // PH_ATTN: 1 = cached K / V travel through the ring (st_attn_ring_ok), 0 = read from global memory (attn_body)
  MVParams mv;      // PH_MATVEC
  AttnParams at;    // PH_ATTN
  EmbedParams em;   // PH_EMBED
  PickParams pk;    // PH_PICK
  XchgParams xc;    // PH_MATVEC with xc.world > 1: the tensor-parallel exchange in front of this phase's staging
};

struct StepArgs {
  const Phase* prog;
  int n_phases;
  int n_slots;
  unsigned* sync;   // [0] grid-barrier arrivals, [1] finished CTAs (the last one resets both), [2] tensor-parallel exchanges done so far
  const int* bounds;   // [n_phases][grid + 1]: first tile of every CTA per mat-vec phase (TileSpace::boundary, computed once on the host)
  unsigned long long* trace;   // optional: per phase and CTA 8 globaltimer stamps {phase starts, input staged, first item ready, phase done,
                               //           previous phase left (barrier entered), arrive issued, all arrived seen, acquire fence done}
};

__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// what lane j knows about tile T0 + j of this CTA's range
struct TileInfo { int seg, til, nch, type; };
template <bool Q3>
__device__ __forceinline__ TileInfo tile_info(const TileSpace& ts, const MVParams& p, int tile, int nb, bool valid) {
  TileInfo ti;
  ti.seg = 0; ti.til = 0; ti.nch = 0; ti.type = GT_Q4_K;
  if (valid) {
    int tl = tile;
    ti.seg = ts.locate(tl);
    ti.til = tl;
    ti.type = ti.seg == 0 ? p.seg[0].w.type : (ti.seg == 1 ? p.seg[1].w.type : p.seg[2].w.type);
    ti.nch = st_chunks<Q3>(ti.type, nb);
  }
  return ti;
}

// source and bytes of work item (chunk kc of tile til) of segment seg, whose type is `type`
struct StItem { const uint8_t* src; uint32_t bytes; };
template <bool Q3>
__device__ __forceinline__ StItem st_item(const MVParams& p, int seg, int type, int til, int kc, int nb) {
  const int kb = st_chunk_blocks<Q3>(type), bb = st_block_bytes<Q3>(type);
  const int nblk = min(kb, nb - kc * kb);
  const uint8_t* base = seg == 0 ? p.seg[0].w.st : (seg == 1 ? p.seg[1].w.st : p.seg[2].w.st);
  return {base + ((size_t)til * nb + (size_t)kc * kb) * bb, (uint32_t)(nblk * bb)};
}

// ---------------------------------------------------------------------------------------------
// Attention phase.  The cached K rows and V channels a task needs are constants of the step (every position but the current
// one was written by earlier launches), so they travel through the SAME ring as the weights: the producer queues them between
// the QKV mat-vec's items and the output projection's, and by the time the grid barrier after QKV opens they sit in shared
// memory.  What is left on the critical path is one L2 round trip for q/k/v, one for the exp table, and arithmetic.
//   K item  up to rows_per_item consecutive cached rows of the task's KV head (head-major cache: one contiguous bulk copy;
//           rows_per_item = ST_SLOT / the padded row's bytes, e.g. 36 rows at hd 128, 44 at hd 100)
//   V item  cv of the task's channels, nchv 256-position chunks each (one bulk copy per channel).  A head's last channel
//           group may hold fewer than ATTN_CH channels, and then fewer items (attn_ring_nv).
struct AttnRingV { int nchv, cv, n_v; };   // V items of a task over T > 0 positions (the host asks for T = n_ctx)
__host__ __device__ inline AttnRingV attn_ring_v(int T) {
  AttnRingV v;
  v.nchv = (T + 255) >> 8;
  v.cv = max(1, min(8, ST_SLOT / (v.nchv * 512)));
  v.n_v = (ATTN_CH + v.cv - 1) / v.cv;
  return v;
}
struct AttnRing : AttnPos, AttnRingV { int n_k, rpi; };
template <bool GEN>
__device__ __forceinline__ AttnRing attn_ring_geom(const AttnParams& p) {
  AttnRing g;
  static_cast<AttnPos&>(g) = attn_pos(p, p.state);
  g.rpi = ST_SLOT / ((GEN ? k_stride(p.hd) : p.hd) * 2);
  if (g.T == 0) { g.n_k = 0; g.n_v = 0; g.cv = 1; g.nchv = 0; return g; }
  static_cast<AttnRingV&>(g) = attn_ring_v(g.T);
  g.n_k = (g.pos + g.rpi - 1) / g.rpi;
  return g;
}
// channels of channel group cg of a head, and the V items they take (g.n_v for a whole group)
__device__ __forceinline__ int attn_group_ch(int hd, int cg) { return min(ATTN_CH, hd - cg * ATTN_CH); }
template <bool GEN>
__device__ __forceinline__ int attn_ring_nv(const AttnRing& g, int hd, int cg) { return GEN && g.n_v > 0 ? (attn_group_ch(hd, cg) + g.cv - 1) / g.cv : g.n_v; }

// producer side of one attention phase (whole warp: lane i issues item i of a task's K run / V groups)
template <bool GEN>
__device__ __forceinline__ void st_attn_produce(const AttnParams& p, uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar, uint32_t S, uint32_t& seq) {
  const int lane = threadIdx.x & 31;
  const AttnRing g = attn_ring_geom<GEN>(p);
  const int n_cg = GEN ? attn_groups(p.hd) : p.hd / ATTN_CH, n_tasks = p.n_head * n_cg, group = p.n_head / p.n_kv, row_bytes = (GEN ? k_stride(p.hd) : p.hd) * 2;
  for (int task = blockIdx.x; task < n_tasks; task += gridDim.x) {
    const int h = task / n_cg, cg = task % n_cg, kvh = h / group;
    const int step = min(32, ST_W * (int)S);   // lanes of one batch never share a slot (see st_producer)
    for (int i0 = 0; i0 < g.n_k; i0 += step) {
      const int i = i0 + lane;
      if (lane < step && i < g.n_k) {
        const uint32_t n = seq + (uint32_t)i;
        const RingPos rp = st_ring(n, S);
        const int rows = min(g.rpi, g.pos - i * g.rpi);
        mbar_wait(&empty_bar[rp.slot], rp.parity ^ 1u, W_FREE_K_SLOT, (int)n);
        mbar_expect_tx(&full_bar[rp.slot], (uint32_t)(rows * row_bytes));
        bulk_g2s(ring + (size_t)rp.slot * ST_SLOT, p.kc + k_row<GEN>(kvh, i * g.rpi, p.n_ctx, p.hd), (uint32_t)(rows * row_bytes), &full_bar[rp.slot]);
      }
      __syncwarp();
    }
    seq += (uint32_t)g.n_k;
    const int n_v = attn_ring_nv<GEN>(g, p.hd, cg), ch_g = GEN ? attn_group_ch(p.hd, cg) : ATTN_CH;
    for (int iv = lane; iv < n_v; iv += 32) {   // n_v <= 32 / cv <= S is checked on the host (st_attn_ring_ok)
      const uint32_t n = seq + (uint32_t)iv;
      const RingPos rp = st_ring(n, S);
      const int nch = min(g.cv, ch_g - iv * g.cv);
      const uint32_t bytes = (uint32_t)(g.nchv * 512);
      mbar_wait(&empty_bar[rp.slot], rp.parity ^ 1u, W_FREE_V_SLOT, (int)n);
      mbar_expect_tx(&full_bar[rp.slot], bytes * nch);
      for (int q = 0; q < nch; q++)
        bulk_g2s(ring + (size_t)rp.slot * ST_SLOT + (size_t)q * bytes, p.vc + v_chan(kvh, cg * ATTN_CH + iv * g.cv + q, p.n_ctx, p.hd), bytes,
                 &full_bar[rp.slot]);
    }
    __syncwarp();
    seq += (uint32_t)n_v;
  }
}

// consumer side: one (head, channel group) task, K / V of the older positions read from the ring, this position's from k16 / v16
template <bool GEN>
__device__ __forceinline__ void st_attn_task(const AttnParams& p, uint8_t* smem, const uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar, uint32_t S, uint32_t seq0,
                                             const AttnRing& g, int h, int cg, float* red_f, double* red_d) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nch = GEN ? attn_group_ch(p.hd, cg) : ATTN_CH;
  const AttnScratch s = attn_scratch<GEN>(smem, p.n_ctx, p.hd, true);
  attn_stage<ST_NT, GEN>(p, s, 0, h, cg, g.pos, attn_cs0<ST_NT>(p, g.pos));
  bar_sync<ST_BAR, ST_NT>();
  // ---- scores: K item i = ring item seq0 + i belongs to warp (seq0 + i) % ST_W (which also frees its slot)
  for (int i = (int)(((uint32_t)warp + ST_W - seq0 % ST_W) % ST_W); i < g.n_k; i += ST_W) {
    const uint32_t n = seq0 + (uint32_t)i;
    const RingPos rp = st_ring(n, S);
    const int r0 = i * g.rpi;
    mbar_wait(&full_bar[rp.slot], rp.parity, W_K_ITEM, (int)n);
    attn_scores<GEN>(p.hd, (const uint16_t*)(ring + (size_t)rp.slot * ST_SLOT), min(g.rpi, g.pos - r0), 0, 8, s.q16, p.kq_scale, s.sc + r0);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[rp.slot]);
  }
  if (warp == (int)((seq0 + (uint32_t)g.n_k) % ST_W)) attn_scores<GEN>(p.hd, s.k16, 1, 0, 8, s.q16, p.kq_scale, s.sc + g.pos);   // the current position
  bar_sync<ST_BAR, ST_NT>();
  attn_softmax<ST_NT, ST_BAR>(s.sc, s.p16, g.T, p.exp_tab, red_f, red_d);
  // ---- V·P for this task's channels
  for (int cc = warp; cc < nch; cc += ST_W) {
    const int c = cg * ATTN_CH + cc;
    const uint32_t n = seq0 + (uint32_t)(g.n_k + cc / g.cv);
    const RingPos rp = st_ring(n, S);
    mbar_wait(&full_bar[rp.slot], rp.parity, W_V_ITEM, (int)n);
    const uint16_t* vrow = (const uint16_t*)(ring + (size_t)rp.slot * ST_SLOT + (size_t)(cc % g.cv) * g.nchv * 512);
    const float o = attn_vp(vrow, s.p16, g, g.pos, s.v16[c]);
    if (lane == 0) p.out[(size_t)h * p.hd + c] = o;
  }
  bar_sync<ST_BAR, ST_NT>();
  if ((int)threadIdx.x < attn_ring_nv<GEN>(g, p.hd, cg)) {
    const uint32_t n = seq0 + (uint32_t)(g.n_k + threadIdx.x);
    mbar_arrive(&empty_bar[st_ring(n, S).slot]);
  }
}

// The consumers' side of an attention phase: tasks (head, channel group) blockIdx.x, + gridDim.x, ...; K / V through the ring
// (ph.q6) or from global memory.  hd 64 / 128 inline (GEN = false), other head sizes in one out-of-line call.
template <bool GEN>
__device__ __forceinline__ void st_attn_phase(const Phase& ph, uint8_t* act_smem, uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar, int n_slots,
                                              uint32_t& seq, float* pick_v, double* red) {
  const int n_cg = GEN ? attn_groups(ph.at.hd) : ph.at.hd / ATTN_CH, n_tasks = ph.at.n_head * n_cg, G = (int)gridDim.x;
  if (ph.q6) {
    const AttnRing ag = attn_ring_geom<GEN>(ph.at);
    for (int task = blockIdx.x; task < n_tasks; task += G) {
      if (task != (int)blockIdx.x) bar_sync<ST_BAR, ST_NT>();
      if (ag.T > 0) st_attn_task<GEN>(ph.at, act_smem, ring, full_bar, empty_bar, (uint32_t)(n_slots / ST_W), seq, ag, task / n_cg, task % n_cg, pick_v, red);
      seq += (uint32_t)(ag.n_k + attn_ring_nv<GEN>(ag, ph.at.hd, task % n_cg));
    }
  } else {
    for (int task = blockIdx.x; task < n_tasks; task += G) {
      if (task != (int)blockIdx.x) bar_sync<ST_BAR, ST_NT>();
      attn_body<ST_NT, ST_BAR, false, GEN>(ph.at, act_smem, task / n_cg, 0, task % n_cg, ph.at.state);
    }
  }
}
// (one copy per kernel build, Q3 and PAIR: ptxas fits an out-of-line function's registers to all its callers at once)
template <bool Q3, bool PAIR>
static __device__ __noinline__ uint32_t st_attn_phase_gen(const Phase& ph, uint8_t* act_smem, uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar, int n_slots,
                                                   uint32_t seq, float* pick_v, double* red) {
  st_attn_phase<true>(ph, act_smem, ring, full_bar, empty_bar, n_slots, seq, pick_v, red);
  return seq;
}

// Producer warp: the same enumeration as the consumers, one bulk copy per item, as far ahead as the ring allows.  The weight
// copies read with an L2 evict-first policy: a weight line is dead once its ring copy has read it (the next read is a step
// later, 4 GB of stream away), so the stream's lines go first and the step's live data (KV cache, activation vectors, exp
// table) stays in L2.  K / V items keep the default policy.
template <bool XC, bool GEN, bool Q3>
__device__ __forceinline__ void st_producer(const StepArgs& args, uint8_t* ring, uint64_t* full_bar, uint64_t* empty_bar) {
  const int lane = threadIdx.x & 31;
  const uint32_t S = (uint32_t)(args.n_slots / ST_W);   // ring depth per consumer warp
  const uint64_t weight_pol = l2_policy_evict_first();
  uint32_t seq = 0;
  for (int ip = 0; ip < args.n_phases; ip++) {
    const Phase* ph = args.prog + ip;
    if (ph->kind == PH_ATTN) {
      if (ph->q6) {
        if (GEN) st_attn_produce<true>(ph->at, ring, full_bar, empty_bar, S, seq);
        else st_attn_produce<false>(ph->at, ring, full_bar, empty_bar, S, seq);
      }
      continue;
    }
    if (ph->kind != PH_MATVEC) continue;
    const MVParams& p = ph->mv;
    TileSpace ts;
    ts.init<Q3>(p);
    const int* bnd = args.bounds + (size_t)ip * (gridDim.x + 1) + blockIdx.x;
    const int T0 = __ldg(bnd), T1 = __ldg(bnd + 1);
    const int nb = p.K >> 8;
    for (int w0 = T0; w0 < T1; w0 += ST_MAXT) {
      const int ntw = min(ST_MAXT, T1 - w0);
      const TileInfo ti = tile_info<Q3>(ts, p, w0 + lane, nb, lane < ntw);
      for (int kc = 0;; kc++) {
        const unsigned mask = __ballot_sync(0xffffffffu, kc < ti.nch);
        if (!mask) break;
        // the items of this row are independent: every lane issues the copy of its own tile (a single issuing thread would cap
        // the stream at one item per ~400 cycles — measured: exactly the 22 B/clk/SM the first build streamed at)
        const int rank = __popc(mask & ((1u << lane) - 1u)), cnt = __popc(mask);
        // at most S lanes at a time: two items of one batch never share a slot, so no lane waits for a slot that only another
        // lane of the same (converged) warp could fill
        for (int base = 0; base < cnt; base += ST_W * (int)S) {
          if (((mask >> lane) & 1u) && rank >= base && rank < base + ST_W * (int)S) {
            const uint32_t n = seq + (uint32_t)rank;
            const RingPos rp = st_ring(n, S);
            const StItem it = st_item<Q3>(p, ti.seg, ti.type, ti.til, kc, nb);
            mbar_wait(&empty_bar[rp.slot], rp.parity ^ 1u, W_FREE_WEIGHT_SLOT, (int)n);
            mbar_expect_tx(&full_bar[rp.slot], it.bytes);
            bulk_g2s_hint(ring + (size_t)rp.slot * ST_SLOT, it.src, it.bytes, &full_bar[rp.slot], weight_pol);
          }
          __syncwarp();
        }
        __syncwarp();
        seq += (uint32_t)__popc(mask);
      }
    }
  }
}

// Consumer side of one mat-vec phase.  `seq` is the running item number (identical in every warp and in the producer).
// XC: the build of the kernel that can exchange partial vectors between ranks (tensor-parallel mode); the single-GPU build
// carries none of that code.  Q3: the build for programs that hold Q3_K matrices (the others carry none of its code).
// PAIR: the build launched as clusters of two CTAs, which stage the input together (stage_q8k_pair).
template <bool XC, bool Q3, bool PAIR>
__device__ __forceinline__ void st_matvec_phase(const Phase& ph, const NormPre& np, uint8_t* ring, uint8_t* act_smem, double* red, uint64_t* full_bar, uint64_t* empty_bar,
                                                float (*mailbox)[ST_STATE * 32], int* flags, uint32_t S, uint32_t& seq, const int* tb, unsigned long long* tr,
                                                unsigned xc_base, PairX& px) {
  const MVParams& p = ph.mv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned epoch = XC ? xc_epoch(xc_base, ph.xc.index) : 0u;   // number of the exchange this phase consumes / produces (if any)
  if constexpr (PAIR) stage_q8k_pair<ST_NT, ST_BAR>(p, np, act_smem, red, px, blockIdx.x < 2);
  else stage_activation<ST_NT, ST_BAR, XC>(p, np, ACT_Q8_K, act_smem, red, blockIdx.x == 0, epoch);
  StAct a = st_act_extras<ST_NT, ST_BAR>(act_smem, p.K, ph.q6 != 0);
  a.xc = XC && ph.xc.role == 2 ? &ph.xc : nullptr;
  a.epoch = epoch;
  if (tr && threadIdx.x == 0) tr[1] = globaltimer_ns();
  bool first_item = tr != nullptr && threadIdx.x == 0;
  TileSpace ts;
  ts.init<Q3>(p);
  const int nb = p.K >> 8;
  const int T0 = tb[0], T1 = tb[1];
#pragma unroll 1
  for (int w0 = T0; w0 < T1; w0 += ST_MAXT) {
    if (w0 != T0) {   // the mailboxes are re-used by the next ST_MAXT tiles
      bar_sync<ST_BAR, ST_NT>();
      if (threadIdx.x < ST_MAXT) flags[threadIdx.x] = 0;
      bar_sync<ST_BAR, ST_NT>();
    }
    const int ntw = min(ST_MAXT, T1 - w0);
    const TileInfo ti = tile_info<Q3>(ts, p, w0 + lane, nb, lane < ntw);
#pragma unroll 1
    for (int kc = 0;; kc++) {
      const unsigned mask = __ballot_sync(0xffffffffu, kc < ti.nch);
      if (!mask) break;
      const int cnt = __popc(mask);
#pragma unroll 1
      for (int r = (int)(((uint32_t)warp + ST_W - seq % ST_W) % ST_W); r < cnt; r += ST_W) {
        unsigned mr = mask;                       // the r-th set bit of mask = the tile (lane) of this item
        for (int q = 0; q < r; q++) mr &= mr - 1;
        const int j = __ffs(mr) - 1;
        const int seg = __shfl_sync(0xffffffffu, ti.seg, j), til = __shfl_sync(0xffffffffu, ti.til, j), type = __shfl_sync(0xffffffffu, ti.type, j);
        const int nch = __shfl_sync(0xffffffffu, ti.nch, j);
        const uint32_t n = seq + (uint32_t)r;
        const RingPos rp = st_ring(n, S);
        const int kb = st_chunk_blocks<Q3>(type);
        const int b0 = kc * kb, nblk = min(kb, nb - b0);
        const MVSeg& sg = p.seg[seg];
        const uint8_t* sp = ring + (size_t)rp.slot * ST_SLOT;
        mbar_wait(&full_bar[rp.slot], rp.parity, W_WEIGHT_ITEM, (int)n);
        if (first_item) { tr[2] = globaltimer_ns(); first_item = false; }
        volatile float* mail = mailbox[j];
        volatile int* flag = flags + j;
        const bool last = kc == nch - 1;
        if (type == GT_Q4_K) run_item<GT_Q4_K, XC>(sp, &empty_bar[rp.slot], nblk, b0, kc, last, a, lane, mail, flag, sg, p, til * ST_ROWS);
        else if (type == GT_Q6_K) run_item<GT_Q6_K, XC>(sp, &empty_bar[rp.slot], nblk, b0, kc, last, a, lane, mail, flag, sg, p, til * ST_ROWS);
        else if (Q3 && type == GT_Q3_K) run_item<GT_Q3_K, XC>(sp, &empty_bar[rp.slot], nblk, b0, kc, last, a, lane, mail, flag, sg, p, til * ST_ROWS);
        else run_item<GT_Q5_K, XC>(sp, &empty_bar[rp.slot], nblk, b0, kc, last, a, lane, mail, flag, sg, p, til * ST_ROWS);
      }
      seq += (uint32_t)cnt;
    }
  }
}

// greedy pick + state advance (k_argmax + k_advance of the un-fused path), CTA 0 only
__device__ __forceinline__ void st_pick_phase(const PickParams& pk, float* bv, int* bi) {
  float best;
  int idx;
  block_argmax<ST_NT, ST_BAR, true>(pk.logits, pk.n, bv, bi, best, idx);
  if (threadIdx.x == 0) {
    pk.state[4] = idx;   // state = {token, position, step, n_total, pick}
    advance_state(pk.state, pk.out_tokens, idx);
  }
}

// End of a persistent launch, after the CTA's last barrier: the last CTA to get here re-arms the grid-barrier words for the
// next launch (sync[0] arrivals, sync[1] finished CTAs) and, when set_xc, stores the tensor-parallel exchange count in sync[2].
__device__ __forceinline__ void grid_rearm(unsigned* sync, bool set_xc = false, unsigned xc = 0) {
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(sync + 1, 1u) == gridDim.x - 1) {
      sync[0] = 0u;
      sync[1] = 0u;
      if (set_xc) sync[2] = xc;
      __threadfence();
    }
  }
}

// GEN: the program's attention phases have a head size other than 64 / 128 (attn_fast_hd); they run in one out-of-line call,
// and the kernels of the other models (GEN = false) have no trace of them.  The tensor-sharded mode takes heads of 64 / 128
// only, so there is no exchange kernel with GEN.  Q3: some phase of the program holds a Q3_K matrix or embedding table.  The
// builds without it compile to the same instructions as before Q3_K was added; with the Q3_K code inlined into every build,
// ptxas spilled more in the builds of the other models (DESIGN.md §6).  PAIR: launched as clusters of two CTAs, which
// stage every mat-vec input together (stage_q8k_pair); the builds without it carry none of that code.  The exchange build
// (XC) is never paired: its staging sums the peers' partial vectors and CTA 0 alone writes sum_out.
template <bool XC, bool GEN, bool Q3, bool PAIR = false>
static __global__ void __launch_bounds__(ST_THREADS, 1) k_step(const __grid_constant__ StepArgs args) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ __align__(8) uint64_t full_bar[ST_MAX_SLOTS];
  __shared__ __align__(8) uint64_t empty_bar[ST_MAX_SLOTS];
  __shared__ double red[3 * ST_W];
  __shared__ __align__(16) float mailbox[ST_MAXT][ST_STATE * 32];
  __shared__ int flags[ST_MAXT];
  __shared__ float pick_v[ST_W];
  __shared__ int pick_i[ST_W];
  __shared__ __align__(16) Phase ph_s[2];   // this phase's descriptor and the next one's (fetched with cp.async a phase ahead)
  __shared__ int tb_s[2][2];                // first / end tile of this CTA, same double buffering
  __shared__ __align__(8) uint64_t pair_bar[PAIR ? 2 : 1];    // PAIR: the exchange rounds of stage_q8k_pair (PairX)
  __shared__ double pair_red[PAIR ? 2 * 2 * 3 * ST_W : 1];
  const int warp = threadIdx.x >> 5;
  uint8_t* ring = smem;
  uint8_t* act_smem = smem + (size_t)args.n_slots * ST_SLOT;
  ring_init(full_bar, empty_bar, args.n_slots, 1);
  PairX px{pair_bar, pair_red, 0u, 0u};
  if constexpr (PAIR) {
    if (threadIdx.x == 0) {
      mbar_init(&pair_bar[0], 1);
      mbar_init(&pair_bar[1], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    px.rank = cluster_ctarank();
    // both CTAs' mbarriers are initialised before either CTA arrives on the other's
    asm volatile("barrier.cluster.arrive.release.aligned;\n barrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
  pdl_trigger();
  pdl_wait();           // (the producer reads device state too: the position decides how many K / V items an attention phase has)
  if (warp == ST_W) {
    st_producer<XC, GEN, Q3>(args, ring, full_bar, empty_bar);
    return;
  }
  const unsigned G = gridDim.x;
  uint32_t seq = 0;
  const unsigned xc_base = XC ? ld_relaxed_u32(args.sync + 2) : 0u;   // (changes only after every CTA has left its last barrier)
  unsigned xc_done = 0;
  // descriptor of phase ip -> ph_s[ip & 1]; issued one phase ahead so that no global round trip sits on the phase boundary
  auto fetch_phase = [&](int ip) {
    if (ip >= args.n_phases) return;
    const uint4* src = (const uint4*)(args.prog + ip);
    const uint32_t dst = st_smem(&ph_s[ip & 1]);
    const int i = (int)threadIdx.x - 32;
    if (i >= 0 && i < (int)(sizeof(Phase) / 16)) asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(dst + i * 16), "l"(src + i) : "memory");
    if (i >= 64 && i < 66)   // this CTA's tile range of that phase
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(st_smem(&tb_s[ip & 1][i - 64])), "l"(args.bounds + (size_t)ip * (gridDim.x + 1) + blockIdx.x + (i - 64)) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  fetch_phase(0);
#pragma unroll 1
  for (int ip = 0; ip < args.n_phases; ip++) {
    bar_sync<ST_BAR, ST_NT>();                 // every consumer warp is done with the previous phase (its stores are issued)
    unsigned long long* const tr = args.trace ? args.trace + ((size_t)ip * G + blockIdx.x) * 8 : nullptr;
    if (tr && threadIdx.x == 0) tr[4] = globaltimer_ns();
    if (threadIdx.x == 0 && ip > 0) {          // grid barrier: one release-arrive, then relaxed polls
      const unsigned target = (unsigned)ip * G;
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(args.sync) : "memory");
      if (tr) tr[5] = globaltimer_ns();
      bounded_wait([&] { return ld_relaxed_u32(args.sync) >= target; }, W_GRID_BARRIER, ip);
      if (tr) { tr[6] = globaltimer_ns(); tr[7] = tr[6]; }
      // no acquire fence: everything the other CTAs produced is read with ld.global.cg (L2, never a stale L1 line), and those
      // loads are issued after the CTA barrier below, i.e. after this poll has returned
    } else {
      asm volatile("cp.async.wait_all;" ::: "memory");
      if (threadIdx.x >= 32 && threadIdx.x < 32 + ST_MAXT) flags[threadIdx.x - 32] = 0;   // (thread 0 is busy with the grid barrier)
    }
    bar_sync<ST_BAR, ST_NT>();
    const Phase& ph = ph_s[ip & 1];
    fetch_phase(ip + 1);
    NormPre np;
    if (ph.kind == PH_MATVEC) preload_norm(np, ph.mv, PAIR ? pair_block0(ph.mv.K >> 8, (int)px.rank) * 256 : 0);
    if (tr && threadIdx.x == 0) tr[0] = globaltimer_ns();
    if (XC && ph.kind == PH_MATVEC && ph.xc.role == 1) xc_done++;
    if (ph.kind == PH_MATVEC) {
      // (the tile bounds were written by threads 0/1 above; the barriers inside the activation staging order them)
      st_matvec_phase<XC, Q3, PAIR>(ph, np, ring, act_smem, red, full_bar, empty_bar, mailbox, flags, (uint32_t)(args.n_slots / ST_W), seq, &tb_s[ip & 1][0], tr,
                                    xc_base, px);
    } else if (ph.kind == PH_ATTN) {
      if (GEN) seq = st_attn_phase_gen<Q3, PAIR>(ph, act_smem, ring, full_bar, empty_bar, args.n_slots, seq, pick_v, red);
      else st_attn_phase<false>(ph, act_smem, ring, full_bar, empty_bar, args.n_slots, seq, pick_v, red);
    } else if (ph.kind == PH_EMBED) {
      if (blockIdx.x == 0) embed_row<Q3>(ph.em, ph.em.tokens[0], ph.em.out, threadIdx.x, ST_NT);
    } else if (ph.kind == PH_PICK) {
      if (blockIdx.x == 0) st_pick_phase(ph.pk, pick_v, pick_i);
    }
    if (tr) {
      bar_sync<ST_BAR, ST_NT>();
      if (threadIdx.x == 0) tr[3] = globaltimer_ns();
    }
  }
  bar_sync<ST_BAR, ST_NT>();
  grid_rearm(args.sync, XC, xc_base + xc_done);
}

// ---------------------------------------------------------------------------------------------
// Host side
struct StepLaunch { int grid; int n_slots; size_t smem; bool gen = false, q3 = false, pair = false; /* k_step<.., GEN, Q3, PAIR>: see k_step */ };

// shared-memory budget: ring slots fill what the largest activation image of the program leaves
inline StepLaunch step_launch_shape(const Phase* phases, int n, int n_sm, size_t max_dyn_smem, size_t extra_act = 0) {
  size_t act = extra_act;
  for (int i = 0; i < n; i++) {
    if (phases[i].kind == PH_MATVEC) act = std::max(act, st_act_bytes(phases[i].mv.K, phases[i].q6 != 0));
    if (phases[i].kind == PH_ATTN) act = std::max(act, attn_smem_bytes(phases[i].at.n_ctx, phases[i].at.hd));
  }
  bool gen = false, q3 = false;
  for (int i = 0; i < n; i++) {
    gen |= phases[i].kind == PH_ATTN && !attn_fast_hd(phases[i].at.hd);
    if (phases[i].kind == PH_MATVEC)
      for (int s = 0; s < phases[i].mv.nseg; s++) q3 |= phases[i].mv.seg[s].w.type == GT_Q3_K;
    q3 |= phases[i].kind == PH_EMBED && phases[i].em.type == GT_Q3_K;
  }
  act = (act + 127) & ~(size_t)127;
  StepLaunch L;
  L.grid = n_sm;
  L.gen = gen;
  L.q3 = q3;
  if (act + (size_t)ST_W * ST_SLOT > max_dyn_smem) { L.n_slots = 0; L.smem = 0; return L; }
  L.n_slots = ST_W * (int)std::min<size_t>(ST_MAX_DEPTH, (max_dyn_smem - act) / ((size_t)ST_W * ST_SLOT));   // whole sub-rings only
  L.smem = (size_t)L.n_slots * ST_SLOT + act;
  return L;
}

// first tile of every CTA for every phase of a program, [n][grid + 1] (the device reads it instead of redoing the 64-bit divisions)
inline std::vector<int> step_bounds(const Phase* phs, int n, int grid) {
  std::vector<int> b((size_t)n * (grid + 1), 0);
  for (int i = 0; i < n; i++) {
    if (phs[i].kind != PH_MATVEC) continue;
    TileSpace ts;
    ts.init(phs[i].mv);
    for (int c = 0; c <= grid; c++) b[(size_t)i * (grid + 1) + c] = ts.boundary(c, grid);
  }
  return b;
}

// can the attention phases of a model with this context feed K / V through a ring of n_slots slots?  A task holds all its V
// items until it ends (its K items are released one by one), so they must fit beside a couple of slots of slack.
inline bool st_attn_ring_ok(int n_ctx, int n_slots) { return attn_ring_v(n_ctx).n_v <= n_slots; }

// a mat-vec phase the step kernel can run: all matrices K-quant (→ Q8_K activations), K a multiple of 256
inline bool step_supports(const MVParams& p) {
  if (p.K % 256) return false;
  for (int s = 0; s < p.nseg; s++)
    if (!type_is_kquant(p.seg[s].w.type) || !p.seg[s].w.st) return false;
  return p.nseg >= 1;
}
inline Phase matvec_phase(const MVParams& p) {
  Phase ph{};
  ph.kind = PH_MATVEC;
  ph.mv = p;
  ph.mv.act = ACT_Q8_K;
  for (int s = 0; s < p.nseg; s++) ph.q6 |= p.seg[s].w.type == GT_Q6_K || p.seg[s].w.type == GT_Q3_K;
  return ph;
}

// point the kernels' watchdog at 4 ints of host-mapped memory (each translation unit has its own copy of the symbol)
static inline cudaError_t st_set_debug_words(int* dev_ptr) { return cudaMemcpyToSymbol(g_st_dbg, &dev_ptr, sizeof(int*)); }
static inline cudaError_t step_set_smem_limit(size_t bytes) {
  void (*const kernels[])(StepArgs) = {k_step<false, false, false>, k_step<false, true, false>, k_step<true, false, false>,
                                        k_step<false, false, true>, k_step<false, true, true>, k_step<true, false, true>};
  for (auto k : kernels) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// Programs with Q3_K matrices are never paired: with the paired staging inlined, their builds spilled more than the unpaired
// ones (DESIGN.md §6), so there are no paired Q3 builds.
inline bool step_paired(const StepLaunch& L, bool xchg) { return L.pair && !L.q3 && !xchg; }
using StepKernel = void (*)(StepArgs);
inline StepKernel step_kernel(const StepLaunch& L, bool xchg) {
  if (xchg) return L.q3 ? k_step<true, false, true> : k_step<true, false, false>;
  if (step_paired(L, xchg)) return L.gen ? k_step<false, true, false, true> : k_step<false, false, false, true>;
  return L.q3 ? (L.gen ? k_step<false, true, true> : k_step<false, false, true>) : (L.gen ? k_step<false, true, false> : k_step<false, false, false>);
}

// Can every mat-vec phase of the program be staged by a pair of CTAs?  Rank 0 holds the larger half of the blocks, 16
// elements per thread and group, at most two groups (stage_q8k_pair): K <= 80 blocks = 20480 with 320 consumer threads.
inline bool step_pair_fits(const Phase* phases, int n) {
  for (int i = 0; i < n; i++)
    if (phases[i].kind == PH_MATVEC && pair_block0(phases[i].mv.K >> 8, 1) * 16 > 2 * ST_NT) return false;
  return true;
}

// the environment knob CTB_ST_CLUSTER=0 keeps the step kernel one CTA per cluster
inline bool step_pair_wanted() {
  const char* e = getenv("CTB_ST_CLUSTER");
  return !(e && e[0] == '0');
}

// step_launch_shape with the dynamic shared memory of the builds that may run the program: the paired builds hold the
// exchange state of stage_q8k_pair in static shared memory, so a program that may run paired sizes its ring for them.
inline StepLaunch step_launch_plan(const Phase* phases, int n, int n_sm, size_t extra_act = 0) {
  StepLaunch L = step_launch_shape(phases, n, n_sm, max_dyn_smem(k_step<true, false, false>), extra_act);
  if (!L.q3 && step_pair_wanted())
    L = step_launch_shape(phases, n, n_sm, std::min(max_dyn_smem(k_step<false, false, false, true>), max_dyn_smem(k_step<false, true, false, true>)), extra_act);
  return L;
}

// Launch the step kernel as clusters of two CTAs, which split every activation staging between them (stage_q8k_pair), when
// pairs are wanted, the program has no Q3_K matrix (step_paired), the grid pairs up, the program fits the split, and all
// grid / 2 clusters are resident at once at this shared-memory size: the grid barrier needs every CTA running.  L must come
// from step_launch_plan (possibly with fewer ring slots).  Sets the shared-memory limit of the paired build it chooses.
inline bool step_pair_choose(StepLaunch& L, const Phase* phases, int n) {
  L.pair = false;
  if (!step_pair_wanted() || L.q3 || L.grid % 2 || !step_pair_fits(phases, n)) return false;
  StepLaunch P = L;
  P.pair = true;
  const StepKernel k = step_kernel(P, false);
  auto check = [](cudaError_t e) {   // (the ring was sized for the paired build: a failure here is an error, not a reason to fall back)
    if (e != cudaSuccess) throw std::runtime_error(std::string("pairing the step kernel: ") + cudaGetErrorString(e));
  };
  check(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(L.grid); cfg.blockDim = dim3(ST_THREADS); cfg.dynamicSmemBytes = L.smem;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  int clusters = 0;
  check(cudaOccupancyMaxActiveClusters(&clusters, k, &cfg));
  L.pair = clusters >= L.grid / 2;
  return L.pair;
}

static inline cudaError_t launch_step(const StepLaunch& L, cudaStream_t st, const Phase* d_prog, const int* d_bounds, int n_phases, unsigned* d_sync, bool pdl = false,
                                      unsigned long long* trace = nullptr, bool xchg = false) {
  StepArgs a;
  a.prog = d_prog; a.bounds = d_bounds; a.n_phases = n_phases; a.n_slots = L.n_slots; a.sync = d_sync; a.trace = trace;
  return launch_kernel_cluster(step_kernel(L, xchg), dim3(L.grid), dim3(ST_THREADS), L.smem, st, pdl, step_paired(L, xchg) ? 2u : 1u, a);
}

}  // namespace ctb
