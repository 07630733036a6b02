// Decode-path mat-vec pieces shared by both kernels of the step (sm_90a), BIT-EXACT with the reference's AVX2 CPU build.
//
//   stage_activation<NT, BAR>  the prologue of every mat-vec: RMSNorm / LayerNorm with fp64 reductions + separate weight (+bias)
//                              multiply (ggml.c:10674-10720, 10605-10654) and the activation quantization to Q8_K (K-quants,
//                              k_quants.c:1191-1226), Q8_0 (Q4_0/Q5_0/Q8_0, ggml.c:1232-1268) or Q8_1 (Q4_1/Q5_1, ggml.c:1420-1481)
//                              into shared memory, never HBM
//   k_matvec                   y[M] = W[M,K]·x[K] for the non-K-quant weight types (Q4_0 / Q5_0 / Q8_0 / Q4_1 / Q5_1 / F16 / F32):
//                              one CTA per SM, warp tasks strided over the grid, the reference kernels' lane order restated
//                              (Q4_0 ggml.c:2500-2525 · Q4_1 2770-2803 · Q5_1 3234-3259 · Q8_0 3379-3402 · F16 2392-2426 · F32 2330-2365)
//   store_epilogue             store | + residual (ggml_add, llama.cpp:2415, 2453) | SiLU / GELU fp16 table (ggml.c:3568-3632)
//
// K-quant weights (Q4_K / Q5_K / Q6_K — everything a Q4_K_M / Q5_K_M file multiplies per token) go through the persistent
// step kernel in stream.cuh, which uses stage_activation and store_epilogue from here.
//
// Why exactness matters: the next mat-mul re-quantizes this output to int8; a 1-ulp difference can flip one rounding and the
// logits then differ by ~1e-3 (measured).  HBM traffic per launch = the weight planes once + O(K) activations from L2.
#pragma once
#include "device_types.cuh"
#include "attention.cuh"

namespace ctb {

#ifndef CTB_THREADS
#define CTB_THREADS 512
#endif
constexpr int MV_THREADS = CTB_THREADS;    // one persistent CTA per SM: the activation prologue is paid once per SM
constexpr int MV_WARPS = MV_THREADS / 32;
constexpr int MV_ROWS = 4;   // Q4_0 / Q8_0: rows per warp (one per 8-lane group, in-lane chain)
constexpr int MV_MAX_SEG = 3;

enum : int { NORM_NONE = 0, NORM_RMS = 1, NORM_LAYER = 2 };
enum : int { EPI_STORE = 0, EPI_ADD = 1, EPI_GELU = 2, EPI_ADD2 = 3, EPI_SILU = 4 };   // GELU / SILU: the reference's fp16-table activation of the row value

// Every spin in the persistent kernels is bounded (bounded_wait): a wait that lasts longer than ST_WATCHDOG_NS writes
// {code, CTA, aux, thread} into host-mapped memory and traps — a protocol bug then ends as a launch failure with a message,
// not as a hung GPU.
#ifndef ST_WATCHDOG_NS
#define ST_WATCHDOG_NS 4000000000ull
#endif
#ifndef XC_WATCHDOG_NS
#define XC_WATCHDOG_NS 30000000000ull   // a peer rank may start its launch late (host jitter): 30 s
#endif
// what a timed-out wait was waiting for (the code st_fail records), and the text the host reports for it
enum WaitCode : int {
  W_GRID_BARRIER = 1, W_FOLD_FLAG, W_FREE_WEIGHT_SLOT, W_WEIGHT_ITEM, W_FREE_K_SLOT, W_FREE_V_SLOT, W_K_ITEM, W_V_ITEM, W_XCHG,
  W_PF_GRID_BARRIER, W_PF_FREE_SLOT, W_PF_WEIGHT_ITEM, W_PAIR, W_CODES
};
constexpr const char* WAIT_TEXT[] = {"?", "grid barrier (aux = phase)", "fold hand-off flag (aux = chunk)", "producer: free weight slot (aux = item)",
                                     "consumer: weight item (aux = item)", "producer: free K slot (attention)", "producer: free V slot (attention)",
                                     "consumer: K item (attention)", "consumer: V item (attention)", "tensor-parallel exchange: a peer's element (aux = exchange number)",
                                     "prefill grid barrier (aux = phase)", "prefill producer: free slot (aux = item)", "prefill consumer: weight item (aux = item)",
                                     "cluster peer: its half of the staged input (aux = exchange round)"};
static_assert(sizeof(WAIT_TEXT) / sizeof(WAIT_TEXT[0]) == W_CODES, "one text per wait code");

static __device__ int* g_st_dbg = nullptr;   // set by the host (st_set_debug_words): 4 ints of mapped pinned host memory, or null
static __device__ __noinline__ void st_fail(WaitCode code, int aux) {
  int* d = g_st_dbg;
  if (d) { d[0] = code; d[1] = (int)blockIdx.x; d[2] = aux; d[3] = (int)threadIdx.x; __threadfence_system(); }
  __trap();
}
// spin until done() holds; one try before the timer is read, st_fail(code, aux) once the wait has lasted limit_ns
template <typename Done>
__device__ __forceinline__ void bounded_wait(Done&& done, WaitCode code, int aux, unsigned long long limit_ns = ST_WATCHDOG_NS) {
  if (done()) return;
  const unsigned long long t0 = globaltimer_ns();
  while (!done())
    if (globaltimer_ns() - t0 > limit_ns) st_fail(code, aux);
}

struct MVSeg {
  DevMat w;
  float* out;          // [M]
  const float* res;    // EPI_ADD: out = acc + res; EPI_ADD2: out = (acc + res) + res2
  const float* res2;
  int epi;
};

struct MVParams {
  const float* x;        // [K] f32 input
  const float* x2;       // x_mode 1: second operand
  int x_mode;            // 0: x;  1: x * x2 (ggml_mul of silu(gate) and up, llama.cpp:2438-2443; the SiLU table is applied by the gate rows' epilogue)
                         // 2: x is a uint2 array of {float bits, exchange number} elements (stream.cuh: XchgParams): the input is
                         //    part[0] + part[1] + ... + part[x_parts-1], parts x_stride elements apart, added in that order
                         //    (tensor-parallel partial sums of a row-parallel mat-vec, one per rank; rank 0's carries the
                         //    residual); an element is valid once its number equals the exchange number the caller passes
  int x_parts, x_stride;
  float* sum_out;        // x_mode 2, optional [K]: CTA 0 writes the summed vector (the residual stream of the next block)
  const float* norm_w;   // [K] or null
  const float* norm_b;   // [K] or null (LayerNorm bias)
  float* norm_out;       // optional [K]: CTA 0 writes the normalised vector (result_norm / embeddings)
  float eps;
  int norm_mode;
  int K;
  int act;               // ACT_*
  int nseg;
  MVSeg seg[MV_MAX_SEG];
  const uint16_t* silu_tab;   // 65536-entry fp16 tables built on the host exactly like ggml.c:4319-4333
  const uint16_t* gelu_tab;
};

// ---------------------------------------------------------------------------------------------
// Shared-memory view of the quantized activation vector.
//   Q8_K: qs is stored lane-major per block: byte offset of int8 word (sub-block s, lane l) = ((b*2 + (s>>2))*8 + l)*16 + (s&3)*4,
//         so GPU lane l reads its 8 words of a block with two conflict-free 16-byte loads.  d: per block.  bs: bsums, natural.
//   Q8_0: natural order; d per 32 (already rounded through fp16).
//   Q8_1: natural order; {d, s} float pairs per 32 at d (d[2b] = d, d[2b + 1] = s of block b).
struct ActView {
  const int8_t* qs;
  const float* d;
  const int16_t* bs;
};

__host__ __device__ inline size_t act_smem_bytes(int act, int K) {
  switch (act) {
    case ACT_Q8_K: return (size_t)K + (((size_t)(K / 256) * 4 + 15) & ~(size_t)15) + (size_t)(K / 16) * 2 + 16;
    case ACT_Q8_0: return (size_t)K + (size_t)(K / 32) * 4 + 16;
    case ACT_Q8_1: return (size_t)K + (size_t)(K / 32) * 8 + 16;
    case ACT_F16: return (size_t)K * 2;
    default: return (size_t)K * 4;
  }
}

// bytes reserved for the per-block d values of a Q8_K vector (keeps the bsums that follow 16-byte aligned)
__host__ __device__ inline size_t q8k_d_bytes(int K) { return ((size_t)(K / 256) * 4 + 15) & ~(size_t)15; }

__device__ __forceinline__ ActView act_view(int act, int K, uint8_t* smem) {
  ActView a;
  a.qs = (const int8_t*)smem;
  const size_t off = ((size_t)K + 15) & ~(size_t)15;
  a.d = (const float*)(smem + off);
  a.bs = (const int16_t*)(smem + off + q8k_d_bytes(K));
  return a;
}

__device__ __forceinline__ int q8k_word_offset(int b, int s, int l) { return ((b * 2 + (s >> 2)) * 8 + l) * 16 + (s & 3) * 4; }

// ---------------------------------------------------------------------------------------------
// Prologue pieces.  Every float operation is spelled with explicit-rounding intrinsics so nvcc cannot
// contract a*b+c into an FMA the reference does not perform — and fuses exactly where the reference binary does.

// Whole prologue: normalise + quantize x[K] into shared memory.
// Each thread owns 16 consecutive elements per pass (one bsums group; 16 threads = one Q8_K block, 2 threads = one Q8_0
// block); all global loads of a pass are issued before anything depends on them.
// CG: the data was produced earlier in the SAME kernel by other SMs (persistent step kernel): read it from L2 (ld.global.cg)
template <bool CG = false>
__device__ __forceinline__ void load16(const float* p, int valid, float (&v)[16]) {
  if (valid >= 16) {
    float4 a, b, c, d;
    if (CG) { a = __ldcg((const float4*)p); b = __ldcg((const float4*)p + 1); c = __ldcg((const float4*)p + 2); d = __ldcg((const float4*)p + 3); }
    else { a = __ldg((const float4*)p); b = __ldg((const float4*)p + 1); c = __ldg((const float4*)p + 2); d = __ldg((const float4*)p + 3); }
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    v[8] = c.x; v[9] = c.y; v[10] = c.z; v[11] = c.w; v[12] = d.x; v[13] = d.y; v[14] = d.z; v[15] = d.w;
  } else {
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = e < valid ? (CG ? __ldcg(p + e) : __ldg(p + e)) : 0.f;
  }
}

template <int NT, int BAR>
__device__ __forceinline__ double block_sum_f64(double s, double* red /* [NT / 32] smem */) {
  s = warp_sum(s);
  bar_sync<BAR, NT>();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  bar_sync<BAR, NT>();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < NT / 32; w++) t += red[w];
  return t;
}
// two sums and a maximum at the price of one sum (red: [3 * NT / 32]); the sums are added in the order block_sum_f64 uses
template <int NT, int BAR>
__device__ __forceinline__ void block_sum2_max_f64(double& s, double& a, double& g, double* red) {
  constexpr int NW = NT / 32;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    a += __shfl_xor_sync(0xffffffffu, a, o);
    g = fmax(g, __shfl_xor_sync(0xffffffffu, g, o));
  }
  bar_sync<BAR, NT>();
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = s; red[NW + (threadIdx.x >> 5)] = a; red[2 * NW + (threadIdx.x >> 5)] = g; }
  bar_sync<BAR, NT>();
  s = 0.0;
  a = 0.0;
#pragma unroll
  for (int w = 0; w < NW; w++) { s += red[w]; a += red[NW + w]; g = fmax(g, red[2 * NW + w]); }
}

__device__ __forceinline__ uint32_t pack4(const int* q) {
  return (uint32_t)(q[0] & 0xff) | ((uint32_t)(q[1] & 0xff) << 8) | ((uint32_t)(q[2] & 0xff) << 16) | ((uint32_t)(q[3] & 0xff) << 24);
}

// 16 consecutive input elements with the producer's activation applied: the reference's fp16-table SiLU (ggml.c:3625-3632)
// times the up projection, or the fp16-table GELU (ggml.c:3568-3575) — fused here instead of in the producing kernel so that
// gate and up can be two independent row sets there.
// 16 consecutive {value, number} elements of one rank's partial vector; spins until all carry `epoch`
__device__ __forceinline__ void load16_ll(const uint2* p, unsigned epoch, float (&u)[16]) {
  uint4 q[8];
  bounded_wait([&] {
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(q[j].x), "=r"(q[j].y), "=r"(q[j].z), "=r"(q[j].w) : "l"(p + 2 * j) : "memory");
    }
#pragma unroll
    for (int j = 0; j < 8; j++) ok &= q[j].y == epoch && q[j].w == epoch;
    return ok;
  }, W_XCHG, (int)epoch, XC_WATCHDOG_NS);
#pragma unroll
  for (int j = 0; j < 8; j++) { u[2 * j] = __uint_as_float(q[j].x); u[2 * j + 1] = __uint_as_float(q[j].z); }
}

template <bool XC = false>
__device__ __forceinline__ void load16x(const MVParams& xs, int base, int valid, float (&v)[16], unsigned epoch = 0) {
  if (XC && xs.x_mode == 2) {   // (K is a multiple of 256 and base of 16: a thread's 16 elements are all valid or all past the end)
    if (valid <= 0) {
#pragma unroll
      for (int e = 0; e < 16; e++) v[e] = 0.f;
      return;
    }
    const uint2* ll = (const uint2*)xs.x + (size_t)(epoch & 1u) * xs.x_parts * xs.x_stride;   // the parity half this exchange uses
    load16_ll(ll + base, epoch, v);
    for (int r = 1; r < xs.x_parts; r++) {
      float u[16];
      load16_ll(ll + (size_t)r * xs.x_stride + base, epoch, u);
#pragma unroll
      for (int e = 0; e < 16; e++) v[e] = __fadd_rn(v[e], u[e]);
    }
    return;
  }
  load16<true>(xs.x + base, valid, v);
  if (xs.x_mode == 1) {          // x = silu_table(gate) (applied once, where the gate row was produced); input = x * up (ggml_mul)
    float u[16];
    load16<true>(xs.x2 + base, valid, u);
#pragma unroll
    for (int e = 0; e < 16; e++) v[e] = __fmul_rn(v[e], u[e]);
  }
}

// Norm weight / bias of this thread's first 16 elements: constants of the model, so they are fetched before the kernel waits
// for its predecessor (pdl_wait) and are in registers when the input vector arrives.
// lo: the first element this CTA stages (stage_q8k_pair; 0 otherwise).
struct NormPre { float w0[16], bias0[16]; };
__device__ __forceinline__ void preload_norm(NormPre& np, const MVParams& p, int lo = 0) {
  const int t = lo + (int)threadIdx.x * 16;
  if (p.norm_mode != NORM_NONE && p.norm_w) load16(p.norm_w + t, p.K - t, np.w0);
  if (p.norm_mode != NORM_NONE && p.norm_b) load16(p.norm_b + t, p.K - t, np.bias0);
}

// ---------------------------------------------------------------------------------------------
// Distributed shared memory of a cluster of two CTAs (stage_q8k_pair): a thread stores into the other CTA's shared memory
// through the address mapa gives for the same offset there.
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t dsmem_map(const void* p, uint32_t rank) {
  uint32_t a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(rank));
  return a;
}
__device__ __forceinline__ void dsmem_st_u32(uint32_t a, uint32_t v) { asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void dsmem_st_u16(uint32_t a, uint16_t v) { asm volatile("st.shared::cluster.u16 [%0], %1;" ::"r"(a), "h"(v) : "memory"); }
__device__ __forceinline__ void dsmem_st_f64(uint32_t a, double v) { asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(a), "d"(v) : "memory"); }

// The two CTAs of a pair hand each other data in numbered rounds.  Round r: every thread stores its data into both CTAs, the
// CTA meets at its named barrier, thread 0 arrives (release, cluster scope) on the peer's mbarrier bar[r & 1], and every thread
// waits (acquire, cluster scope) on its own bar[r & 1] for the peer's arrival.  The named barrier orders all of this CTA's
// stores before thread 0's release; each waiting thread's acquire then orders the peer's stores before its own loads.  A CTA
// arrives for round r + 2 only after it has waited for round r + 1, which the peer sends after it has finished waiting for
// round r, so two mbarriers (and two reduction buffers) never hold two rounds at once.  Every round's data lands in a CTA
// that is still waiting for it, so no CTA stores into one that has exited.
struct PairX {
  uint64_t* bar;    // [2] mbarriers of this CTA, arrival count 1 (initialised before the launch's first cluster barrier)
  double* red;      // [2 rounds][2 ranks][3][NT / 32] per-warp partials of the norm statistic
  uint32_t rank;    // %cluster_ctarank
  uint32_t round;   // rounds done so far: the same in both CTAs
};
// blocks [pair_block0(nb, r), pair_block0(nb, r + 1)) of a vector of nb Q8_K blocks are rank r's; an odd block goes to rank 0
__host__ __device__ inline int pair_block0(int nb, int rank) { return rank <= 0 ? 0 : (rank == 1 ? (nb + 1) / 2 : nb); }

template <int NT, int BAR>
__device__ __forceinline__ void pair_round(PairX& px) {
  bar_sync<BAR, NT>();
  uint64_t* bar = px.bar + (px.round & 1u);
  if (threadIdx.x == 0) asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(dsmem_map(bar, px.rank ^ 1u)) : "memory");
  const uint32_t addr = (uint32_t)__cvta_generic_to_shared(bar), parity = (px.round >> 1) & 1u;
  bounded_wait([&] {
    uint32_t ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    return ok != 0;
  }, W_PAIR, (int)px.round);
  px.round++;
}

// block_sum2_max_f64 over both CTAs of the pair: the per-warp partials of both go to both, and every thread adds them in one
// fixed order, rank 0's warps first, so both CTAs hold the same s, a and g.
template <int NT, int BAR>
__device__ __forceinline__ void pair_sum2_max_f64(double& s, double& a, double& g, bool a_is_s, PairX& px) {
  constexpr int NW = NT / 32;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    if (!a_is_s) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      g = fmax(g, __shfl_xor_sync(0xffffffffu, g, o));
    }
  }
  double* buf = px.red + (px.round & 1u) * (2 * 3 * NW);
  if ((threadIdx.x & 31) == 0) {
    const int w = threadIdx.x >> 5;
    double* mine = buf + px.rank * (3 * NW);
    mine[w] = s; mine[NW + w] = a; mine[2 * NW + w] = g;
    const uint32_t peer = dsmem_map(mine, px.rank ^ 1u);
    dsmem_st_f64(peer + 8 * w, s); dsmem_st_f64(peer + 8 * (NW + w), a); dsmem_st_f64(peer + 8 * (2 * NW + w), g);
  }
  pair_round<NT, BAR>(px);
  s = 0.0;
  a = 0.0;
#pragma unroll
  for (int r = 0; r < 2; r++)
#pragma unroll
    for (int w = 0; w < NW; w++) { s += buf[r * 3 * NW + w]; a += buf[r * 3 * NW + NW + w]; g = fmax(g, buf[r * 3 * NW + 2 * NW + w]); }
  if (a_is_s) a = s;
}

// One norm statistic, (float)(Σ term(x_i) / K), as the reference computes it: its double sum runs over the elements one after
// another (ggml.c:10700-10703 / 10630-10645).  The threads add the same terms in another order (16-element chains, the warp
// butterfly, the warps in order), and a double sum of float terms is not exact once they span more than about 53 - 24 -
// log2(K) bits: then the two orders can round the float statistic differently.  Every order of K terms lies within
// γ_K·Σ|t_i| of the exact sum (γ_K = K·u / (1 - K·u), u = 2^-53; an addition of an exact 0 is exact), so the reference's sum
// lies within 2γ_K·A of the parallel one S, with A = Σ|t_i| (from below, A ≥ (1 - γ_K)·A_exact; the factor below covers that
// for K ≤ 2^20).  Division and rounding to float are monotone: when both ends of [S - e, S + e] give the same float, so does
// the reference's sum and S is used.  Otherwise (about K·2^-26 of normalisations by the bound) warp 0 adds the terms in
// element order and broadcasts the sum.  s / a: this thread's partial sums of the terms / of |terms| (a_is_s: the terms are
// never negative, so A = S and a is not reduced).  Every thread, and every CTA, sees the same S and A and takes the same branch.
// LayerNorm's Σx of an input whose mean is near 0 fails the bound (|S| << A) too often; there every term is usually a multiple
// of the smallest term's lsb, 1 / g, and A < 2^52 / g: then no partial sum in any order rounds and S is exact.  g: the largest
// 1 / lsb over this thread's terms (lsb_inv; a_is_s: unused).
__device__ __forceinline__ unsigned min_exp(unsigned emin, float t) {   // smallest exponent field of a non-zero term (subnormal: 1)
  const unsigned bits = __float_as_uint(t) & 0x7fffffffu;
  return bits ? min(emin, max(bits >> 23, 1u)) : emin;
}
__device__ __forceinline__ double lsb_inv(unsigned emin) { return ldexp(1.0, 150 - (int)emin); }

enum : int { NORM_TERM_SQ = 0, NORM_TERM_X = 1, NORM_TERM_DEV = 2 };   // x², x, (x - mean)²
// The statistic's sum in element order, by warp 0: it loads 512 elements at a time and every lane adds all of them.  Out of
// line, one copy for the three statistics: it runs on few normalisations and would otherwise grow every kernel's hot code.
// It takes the input's fields by value, so a caller's MVParams never has to live in local memory for its sake.
template <bool XC>
static __device__ __noinline__ double seq_sum_warp0(const float* x, const float* x2, int x_mode, int x_parts, int x_stride, int K, int kind,
                                                    float mean, unsigned epoch) {
  MVParams xs;
  xs.x = x; xs.x2 = x2; xs.x_mode = x_mode; xs.x_parts = x_parts; xs.x_stride = x_stride;
  const int lane = threadIdx.x & 31;
  double seq = 0.0;
  for (int base = 0; base < K; base += 512) {
    float v[16];
    load16x<XC>(xs, base + lane * 16, K - base - lane * 16, v, epoch);
    for (int l = 0; l < 32; l++)
#pragma unroll
      for (int i = 0; i < 16; i++) {
        float t = __shfl_sync(0xffffffffu, v[i], l);
        if (kind == NORM_TERM_DEV) t = __fsub_rn(t, mean);
        if (base + l * 16 + i < K) seq += kind == NORM_TERM_X ? (double)t : (double)__fmul_rn(t, t);
      }
  }
  return seq;
}

// PAIR: the terms are spread over the two CTAs of a pair (stage_q8k_pair), which add all partial sums in the same order.
template <int NT, int BAR, bool XC, bool PAIR = false>
__device__ __forceinline__ float norm_stat(double s, double a, double g, bool a_is_s, int kind, float mean, const MVParams& xs, double* red,
                                           unsigned epoch, PairX* px = nullptr) {
  const int K = xs.K;
  if constexpr (PAIR) pair_sum2_max_f64<NT, BAR>(s, a, g, a_is_s, *px);
  else if (a_is_s) a = s = block_sum_f64<NT, BAR>(s, red);
  else block_sum2_max_f64<NT, BAR>(s, a, g, red);
  // inf / NaN terms give the same sum in every order (a double sum of float terms cannot overflow); so does an exact sum
  if (!isfinite(s) || (!a_is_s && __dmul_ru(a, g) < 0x1p52)) return (float)(s / (double)K);
  const double e = __dmul_ru(a, (double)K * 0x1.0000001p-52);   // ≥ 2γ_K / (1 - γ_K) · A, rounded up
  const float lo = (float)(__dsub_rd(s, e) / (double)K), hi = (float)(__dadd_ru(s, e) / (double)K);
  if (lo == hi) return lo;
  const double seq = threadIdx.x < 32 ? seq_sum_warp0<XC>(xs.x, xs.x2, xs.x_mode, xs.x_parts, xs.x_stride, K, kind, mean, epoch) : 0.0;
  bar_sync<BAR, NT>();   // every thread has read the partials out of red
  if (threadIdx.x == 0) red[0] = seq;
  bar_sync<BAR, NT>();
  return (float)(red[0] / (double)K);
}

// ggml_rms_norm / ggml_norm of 16 elements given the statistic (mean, scale), then the separate weight and bias (ggml_mul, ggml_add)
__device__ __forceinline__ void norm_apply16(float (&v)[16], const float (&w)[16], const float (&bb)[16], int norm_mode, float mean, float scale, bool has_w,
                                             bool has_b) {
#pragma unroll
  for (int e = 0; e < 16; e++) {
    float y = v[e];
    if (norm_mode == NORM_LAYER) y = __fsub_rn(y, mean);
    y = __fmul_rn(y, scale);
    if (has_w) y = __fmul_rn(y, w[e]);
    if (has_b) y = __fadd_rn(y, bb[e]);
    v[e] = y;
  }
}

// One thread's 16 elements of a Q8_K block (16 lanes, a half-warp, share a block; every lane of the warp calls): reference
// quantize_row_q8_K_reference (k_quants.c:1191-1226): the first element with the largest |x| fixes the sign; iscale = -128/max;
// q = min(127, nearest_int(iscale*x)); the reference BINARY fuses iscale*x + 12582912.f (vfmadd), so the exact product is
// rounded once — __fmaf_rn.  d = 1/iscale; bsums per 16.  PAIR: the same words also go to the other CTA of the pair, whose
// image has the same layout at pqs (qs), pdd (d) and pbs (bsums).
template <bool PAIR = false>
__device__ __forceinline__ void quant_q8k16(const float (&v)[16], int base, int valid, int lane, int8_t* qs, float* dd, int16_t* bs, uint32_t pqs = 0,
                                            uint32_t pdd = 0, uint32_t pbs = 0) {
  float amax = 0.f, mx = 0.f;
#pragma unroll
  for (int e = 0; e < 16; e++) { const float ax = fabsf(v[e]); if (ax > amax) { amax = ax; mx = v[e]; } }
  float gmax = amax;
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
  const unsigned who = __ballot_sync(0xffffffffu, amax == gmax);
  const int hbase = lane & 16, hl = lane & 15;
  const unsigned mine = (who >> hbase) & 0xffffu;
  const float maxv = __shfl_sync(0xffffffffu, mx, hbase + __ffs(mine) - 1);
  if (valid > 0) {
    const int b = base >> 8;
    int q[16];
    int sum = 0;
    if (gmax == 0.f) {
#pragma unroll
      for (int e = 0; e < 16; e++) q[e] = 0;
      if (hl == 0) {
        dd[b] = 0.f;
        if (PAIR) dsmem_st_u32(pdd + 4 * b, 0u);
      }
    } else {
      const float iscale = __fdiv_rn(-128.f, maxv);
#pragma unroll
      for (int e = 0; e < 16; e++) {
        const float val = __fmaf_rn(iscale, v[e], 12582912.f);
        q[e] = min(127, (__float_as_int(val) & 0x007fffff) - 0x00400000);
        sum += q[e];
      }
      if (hl == 0) {
        const float d = __fdiv_rn(1.f, iscale);
        dd[b] = d;
        if (PAIR) dsmem_st_u32(pdd + 4 * b, __float_as_uint(d));
      }
    }
    bs[b * 16 + hl] = (int16_t)sum;
    if (PAIR) dsmem_st_u16(pbs + 2 * (b * 16 + hl), (uint16_t)(int16_t)sum);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int wi = hl * 4 + j, o = q8k_word_offset(b, wi >> 3, wi & 7);
      *(uint32_t*)(qs + o) = pack4(q + 4 * j);
      if (PAIR) dsmem_st_u32(pqs + o, pack4(q + 4 * j));
    }
  }
}

// The first NT threads of the CTA must call (named barrier BAR); each owns 16 consecutive elements per pass.
// red: 3 * NT / 32 doubles of shared memory.
template <int NT, int BAR, bool XC = false>   // XC: the input may be a tensor-parallel exchange (x_mode 2); compiled out otherwise
__device__ __forceinline__ void stage_activation(const MVParams& xs, const NormPre& np, int act, uint8_t* smem, double* red, bool write_norm, unsigned epoch = 0) {
  const float* nw = xs.norm_w;
  const float* nb_ = xs.norm_b;
  float* norm_out = xs.norm_out;
  const int norm_mode = xs.norm_mode, K = xs.K;
  const float eps = xs.eps;
  const int t = threadIdx.x, lane = t & 31;
  const int passes = (K + NT * 16 - 1) / (NT * 16);
  // ---- statistics: fp64 sums, the reference's float result (norm_stat)
  float mean = 0.f, scale = 1.f;
  float v0[16];                          // pass 0's x stays in registers
  load16x<XC>(xs, t * 16, K - t * 16, v0, epoch);
  if (norm_mode == NORM_RMS) {
    double ss = 0.0;
    for (int ps = 0; ps < passes; ps++) {
      const int base = (ps * NT + t) * 16;
      if ((base & ~511) >= K) continue;     // the whole warp lies past the end of x (warp-uniform): nothing to add
      float v[16];
      if (ps == 0) {
#pragma unroll
        for (int e = 0; e < 16; e++) v[e] = v0[e];
      } else load16x<XC>(xs, base, K - base, v, epoch);
#pragma unroll
      for (int e = 0; e < 16; e++) ss += (double)__fmul_rn(v[e], v[e]);
    }
    const float m = norm_stat<NT, BAR, XC>(ss, ss, 0.0, true, NORM_TERM_SQ, 0.f, xs, red, epoch);
    scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(m, eps)));
  } else if (norm_mode == NORM_LAYER) {
    double s1 = 0.0, a1 = 0.0;
    unsigned emin = 255;
    for (int ps = 0; ps < passes; ps++) {
      const int base = (ps * NT + t) * 16;
      if ((base & ~511) >= K) continue;
      float v[16];
      load16x<XC>(xs, base, K - base, v, epoch);
#pragma unroll
      for (int e = 0; e < 16; e++) {
        s1 += (double)v[e];
        a1 += (double)fabsf(v[e]);
        emin = min_exp(emin, v[e]);
      }
    }
    mean = norm_stat<NT, BAR, XC>(s1, a1, lsb_inv(emin), false, NORM_TERM_X, 0.f, xs, red, epoch);
    double s2 = 0.0;
    for (int ps = 0; ps < passes; ps++) {
      const int base = (ps * NT + t) * 16;
      if ((base & ~511) >= K) continue;
      float v[16];
      load16x<XC>(xs, base, K - base, v, epoch);
#pragma unroll
      for (int e = 0; e < 16; e++) { const float d = (base + e < K) ? __fsub_rn(v[e], mean) : 0.f; s2 += (double)__fmul_rn(d, d); }
    }
    const float var = norm_stat<NT, BAR, XC>(s2, s2, 0.0, true, NORM_TERM_DEV, mean, xs, red, epoch);
    scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, eps)));
  }
  // ---- normalise + quantize
  int8_t* qs = (int8_t*)smem;
  const size_t off = ((size_t)K + 15) & ~(size_t)15;
  float* dd = (float*)(smem + off);
  int16_t* bs = (int16_t*)(smem + off + q8k_d_bytes(K));
  for (int ps = 0; ps < passes; ps++) {
    const int base = (ps * NT + t) * 16;
    const int valid = K - base;
    if ((base & ~511) >= K) continue;       // warp-uniform: this warp has no elements in this pass
    float v[16];
    if (ps == 0) {
#pragma unroll
      for (int e = 0; e < 16; e++) v[e] = v0[e];
    } else load16x<XC>(xs, base, valid, v, epoch);
    if (XC && write_norm && xs.x_mode == 2 && xs.sum_out && valid > 0) {
#pragma unroll
      for (int e = 0; e < 16; e++) if (e < valid) xs.sum_out[base + e] = v[e];
    }
    if (norm_mode != NORM_NONE) {
      float w[16], bb[16];
      if (ps == 0) {
#pragma unroll
        for (int e = 0; e < 16; e++) { w[e] = np.w0[e]; bb[e] = np.bias0[e]; }
      } else {
        if (nw) load16(nw + base, valid, w);
        if (nb_) load16(nb_ + base, valid, bb);
      }
      norm_apply16(v, w, bb, norm_mode, mean, scale, nw != nullptr, nb_ != nullptr);
    }
    if (write_norm && norm_out && valid > 0) {
#pragma unroll
      for (int e = 0; e < 16; e++) if (e < valid) norm_out[base + e] = v[e];
    }
    if (act == ACT_Q8_K) {
      quant_q8k16(v, base, valid, lane, qs, dd, bs);
    } else if (act == ACT_Q8_0) {
      // quantize_row_q8_0, AVX2 variant (ggml.c:1232-1268): d = amax/127 kept as fp16, id = 127/amax, round-half-even
      float amax = 0.f;
#pragma unroll
      for (int e = 0; e < 16; e++) amax = fmaxf(amax, fabsf(v[e]));
      amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
      if (valid > 0) {
        const float d = __fdiv_rn(amax, 127.f);
        const float id = amax != 0.f ? __fdiv_rn(127.f, amax) : 0.f;
        int q[16];
#pragma unroll
        for (int e = 0; e < 16; e++) q[e] = __float2int_rn(__fmul_rn(v[e], id));
        *(uint4*)(qs + base) = make_uint4(pack4(q), pack4(q + 4), pack4(q + 8), pack4(q + 12));
        if ((lane & 1) == 0) dd[base >> 5] = h2f(f2h(d));
      }
    } else if (act == ACT_Q8_1) {
      // quantize_row_q8_1, AVX2 variant (ggml.c:1420-1481): as Q8_0, but d = amax/127 stays a float, and s = d * (float)Σq
      // over the block (an exact integer sum; the two threads of a block add their halves)
      float amax = 0.f;
#pragma unroll
      for (int e = 0; e < 16; e++) amax = fmaxf(amax, fabsf(v[e]));
      amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
      const float d = __fdiv_rn(amax, 127.f);
      const float id = amax != 0.f ? __fdiv_rn(127.f, amax) : 0.f;
      int q[16];
      int sum = 0;
#pragma unroll
      for (int e = 0; e < 16; e++) { q[e] = __float2int_rn(__fmul_rn(v[e], id)); sum += q[e]; }
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      if (valid > 0) {
        *(uint4*)(qs + base) = make_uint4(pack4(q), pack4(q + 4), pack4(q + 8), pack4(q + 12));
        if ((lane & 1) == 0) *(float2*)(dd + (base >> 4)) = make_float2(d, __fmul_rn(d, (float)sum));
      }
    } else if (act == ACT_F16) {
      uint16_t* h = (uint16_t*)smem;
#pragma unroll
      for (int e = 0; e < 16; e++) if (e < valid) h[base + e] = f2h(v[e]);
    } else {
      float* f = (float*)smem;
#pragma unroll
      for (int e = 0; e < 16; e++) if (e < valid) f[base + e] = v[e];
    }
  }
  bar_sync<BAR, NT>();
}

// stage_activation's Q8_K staging split over the two CTAs of a cluster (the paired k_step launch, stream.cuh): rank r loads,
// normalises and quantizes the whole blocks [pair_block0(nb, r), pair_block0(nb, r + 1)) and stores them into both CTAs'
// images; the norm statistic's per-warp partials cross over too (pair_sum2_max_f64).  Each block is quantized from the same
// floats by the same code as in stage_activation, and norm_stat gives the reference's float whatever the order of
// the partial sums (its bound holds for every order, and its fallback adds the whole vector in element order), so both images
// are stage_activation's bits.  A thread holds at most two groups of 16 (the host pairs only programs where that suffices:
// step_pair_fits), and both are loaded before either is used.  write_norm: this pair writes norm_out, each rank its blocks.
template <int NT, int BAR>
__device__ __forceinline__ void stage_q8k_pair(const MVParams& xs, const NormPre& np, uint8_t* smem, double* red, PairX& px, bool write_norm) {
  const int K = xs.K, nb = K >> 8, norm_mode = xs.norm_mode, t = threadIdx.x, lane = t & 31;
  const int lo = pair_block0(nb, (int)px.rank) * 256, hi = pair_block0(nb, (int)px.rank + 1) * 256;
  const int base[2] = {lo + t * 16, lo + (t + NT) * 16};
  float v[2][16];   // zeros past hi
  load16x(xs, base[0], hi - base[0], v[0]);
  load16x(xs, base[1], hi - base[1], v[1]);
  // ---- statistics
  float mean = 0.f, scale = 1.f;
  if (norm_mode == NORM_RMS) {
    double ss = 0.0;
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 16; e++) ss += (double)__fmul_rn(v[h][e], v[h][e]);
    const float m = norm_stat<NT, BAR, false, true>(ss, ss, 0.0, true, NORM_TERM_SQ, 0.f, xs, red, 0, &px);
    scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(m, xs.eps)));
  } else if (norm_mode == NORM_LAYER) {
    double s1 = 0.0, a1 = 0.0;
    unsigned emin = 255;
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 16; e++) {
        s1 += (double)v[h][e];
        a1 += (double)fabsf(v[h][e]);
        emin = min_exp(emin, v[h][e]);
      }
    mean = norm_stat<NT, BAR, false, true>(s1, a1, lsb_inv(emin), false, NORM_TERM_X, 0.f, xs, red, 0, &px);
    double s2 = 0.0;
#pragma unroll
    for (int h = 0; h < 2; h++)
      if (base[h] < hi) {
#pragma unroll
        for (int e = 0; e < 16; e++) { const float d = __fsub_rn(v[h][e], mean); s2 += (double)__fmul_rn(d, d); }
      }
    const float var = norm_stat<NT, BAR, false, true>(s2, s2, 0.0, true, NORM_TERM_DEV, mean, xs, red, 0, &px);
    scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, xs.eps)));
  }
  // ---- normalise + quantize into both images
  int8_t* qs = (int8_t*)smem;
  float* dd = (float*)(smem + (((size_t)K + 15) & ~(size_t)15));
  int16_t* bs = (int16_t*)((uint8_t*)dd + q8k_d_bytes(K));
  const uint32_t peer = px.rank ^ 1u, pqs = dsmem_map(qs, peer), pdd = dsmem_map(dd, peer), pbs = dsmem_map(bs, peer);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    if (lo + (((h * NT + t) * 16) & ~511) >= hi) continue;   // warp-uniform: this warp has no elements in this group
    const int valid = hi - base[h];
    if (norm_mode != NORM_NONE) {
      float w[16], bb[16];
      if (h == 0) {
#pragma unroll
        for (int e = 0; e < 16; e++) { w[e] = np.w0[e]; bb[e] = np.bias0[e]; }
      } else {
        if (xs.norm_w) load16(xs.norm_w + base[h], valid, w);
        if (xs.norm_b) load16(xs.norm_b + base[h], valid, bb);
      }
      norm_apply16(v[h], w, bb, norm_mode, mean, scale, xs.norm_w != nullptr, xs.norm_b != nullptr);
    }
    if (write_norm && xs.norm_out && valid > 0) {
#pragma unroll
      for (int e = 0; e < 16; e++) xs.norm_out[base[h] + e] = v[h][e];
    }
    quant_q8k16<true>(v[h], base[h], valid, lane, qs, dd, bs, pqs, pdd, pbs);
  }
  pair_round<NT, BAR>(px);
}

// ---------------------------------------------------------------------------------------------
// hsum_float_8 (ggml.c:609-615) over the 8 lanes of a group: ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7)); every lane ends with the sum.
__device__ __forceinline__ float group_hsum8(float v) {
  v = v + __shfl_xor_sync(0xffffffffu, v, 4);
  v = v + __shfl_xor_sync(0xffffffffu, v, 2);
  v = v + __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}

// Q4_0: natural plane; lane l uses word (l & 3) of the block's 16 nibble bytes, low nibbles for l < 4 (elements 4l..4l+3),
// high nibbles for l >= 4 (elements 16+4(l-4)..).  bytes_from_nibbles_32 - 8, then the s8·s8 dot (ggml.c:2500-2525).
__device__ __forceinline__ float dot_q40(const DevMat& w, int row, const ActView& a, int l) {
  const int nb = w.nb;
  const uint8_t* qrow = w.qs + (size_t)row * nb * 16 + (l & 3) * 4;
  const uint16_t* drow = w.d + (size_t)row * nb;
  const int shift = (l >> 2) * 4;
  float acc = 0.f;
#pragma unroll 8
  for (int b = 0; b < nb; b++) {
    const uint32_t q = (uint32_t)__ldg((const int*)(qrow + (size_t)b * 16));
    const float dw = h2f(__ldg(drow + b));
    const int aw = *(const int*)(a.qs + b * 32 + l * 4);
    const float yd = a.d[b];
    const uint32_t nib = (q >> shift) & 0x0f0f0f0fu;
    const uint32_t bx = ((nib | 0x80808080u) - 0x08080808u) ^ 0x80808080u;   // per-byte (nib - 8), two's complement, no borrow
    acc = __fmaf_rn(__fmul_rn(dw, yd), (float)__dp4a((int)bx, aw, 0), acc);
  }
  return group_hsum8(acc);
}

// Q5_0 (ggml.c:2983-3005): the nibble as for Q4_0 plus the fifth bit from qh (bit j = element j): the AVX2 kernel ORs 0xF0 into
// the bytes whose bit is CLEAR, i.e. the int8 value is q5 - 16; then the same s8·s8 dot, fmadd and hsum as Q4_0.
__device__ __forceinline__ float dot_q50(const DevMat& w, int row, const ActView& a, int l) {
  const int nb = w.nb;
  const uint8_t* qrow = w.qs + (size_t)row * nb * 16 + (l & 3) * 4;
  const uint32_t* hrow = (const uint32_t*)w.qh + (size_t)row * nb;
  const uint16_t* drow = w.d + (size_t)row * nb;
  const int shift = (l >> 2) * 4;
  float acc = 0.f;
#pragma unroll 8
  for (int b = 0; b < nb; b++) {
    const uint32_t q = (uint32_t)__ldg((const int*)(qrow + (size_t)b * 16));
    const uint32_t h4 = (__ldg(hrow + b) >> (4 * l)) & 0xfu;               // fifth bits of elements 4l..4l+3
    const float dw = h2f(__ldg(drow + b));
    const int aw = *(const int*)(a.qs + b * 32 + l * 4);
    const float yd = a.d[b];
    const uint32_t nib = (q >> shift) & 0x0f0f0f0fu;
    const uint32_t set = (h4 * 0x00204081u) & 0x01010101u;                   // bit k of h4 -> bit 0 of byte k
    const uint32_t bx = nib | ((set ^ 0x01010101u) * 0xf0u);                 // per byte: nibble - 16 when the bit is clear
    acc = __fmaf_rn(__fmul_rn(dw, yd), (float)__dp4a((int)bx, aw, 0), acc);
  }
  return group_hsum8(acc);
}

__device__ __forceinline__ float dot_q80(const DevMat& w, int row, const ActView& a, int l) {
  const int nb = w.nb;
  const uint8_t* qrow = w.qs + (size_t)row * nb * 32 + l * 4;
  const uint16_t* drow = w.d + (size_t)row * nb;
  float acc = 0.f;
#pragma unroll 8
  for (int b = 0; b < nb; b++) {
    const int q = __ldg((const int*)(qrow + (size_t)b * 32));
    const float dw = h2f(__ldg(drow + b));
    const int aw = *(const int*)(a.qs + b * 32 + l * 4);
    acc = __fmaf_rn(__fmul_rn(dw, a.d[b]), (float)__dp4a(q, aw, 0), acc);
  }
  return group_hsum8(acc);
}

// Q4_1 / Q5_1 with a Q8_1 activation (ggml.c:2770-2803, 3234-3259): unsigned nibbles (Q5_1: the fifth bit ORed in as 0x10, value
// 0..31), lane l the integer sum of elements 4l..4l+3 (bytes_from_nibbles_32 + mul_sum_us8_pairs_float), acc = fma(d_w*d_y, sum,
// acc) per block; the mins enter through the scalar chain summs += m_w * s_y in block order, which the reference binary fuses
// (vfmadd231ss), and the result is hsum_float_8(acc) + summs.  Every lane of the row's group runs the same summs chain.
template <bool Q5>
__device__ __forceinline__ float dot_q1(const DevMat& w, int row, const ActView& a, int l) {
  const int nb = w.nb;
  const uint8_t* qrow = w.qs + (size_t)row * nb * 16 + (l & 3) * 4;
  const uint32_t* hrow = (const uint32_t*)w.qh + (size_t)row * nb;
  const uint16_t* drow = w.d + (size_t)row * nb;
  const uint16_t* mrow = w.mn + (size_t)row * nb;
  const int shift = (l >> 2) * 4;
  float acc = 0.f, summs = 0.f;
#pragma unroll 8
  for (int b = 0; b < nb; b++) {
    const uint32_t q = (uint32_t)__ldg((const int*)(qrow + (size_t)b * 16));
    const float dw = h2f(__ldg(drow + b));
    const float mw = h2f(__ldg(mrow + b));
    const int aw = *(const int*)(a.qs + b * 32 + l * 4);
    const float2 ds = *(const float2*)(a.d + 2 * b);
    uint32_t bx = (q >> shift) & 0x0f0f0f0fu;
    if (Q5) bx |= ((((__ldg(hrow + b) >> (4 * l)) & 0xfu) * 0x00204081u) & 0x01010101u) << 4;   // bit k of the 4 -> 0x10 in byte k
    acc = __fmaf_rn(__fmul_rn(dw, ds.x), (float)__dp4a((int)bx, aw, 0), acc);
    summs = __fmaf_rn(mw, ds.y, summs);
  }
  return __fadd_rn(group_hsum8(acc), summs);
}

__device__ __forceinline__ float dot_legacy(const DevMat& w, int row, const ActView& a, int l) {
  switch (w.type) {
    case GT_Q4_0: return dot_q40(w, row, a, l);
    case GT_Q5_0: return dot_q50(w, row, a, l);
    case GT_Q4_1: return dot_q1<false>(w, row, a, l);
    case GT_Q5_1: return dot_q1<true>(w, row, a, l);
    default: return dot_q80(w, row, a, l);
  }
}

// GGML_F32x8_REDUCE over a warp that plays 4 accumulators x 8 lanes (lane = 8*j + l): (0+2),(1+3) -> (0+1) -> lo128+hi128 ->
// hadd -> hadd  (ggml.c:1964-1982).  All lanes end with the result.
__device__ __forceinline__ float warp_reduce_f32x8(float v) {
  v = v + __shfl_xor_sync(0xffffffffu, v, 16);
  v = v + __shfl_xor_sync(0xffffffffu, v, 8);
  v = v + __shfl_xor_sync(0xffffffffu, v, 4);
  v = v + __shfl_xor_sync(0xffffffffu, v, 1);
  v = v + __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// F16 weights: ggml_vec_dot_f16 (ggml.c:2392-2426), one warp per row: lane L owns elements 32i+L, one fma per step,
// the reduce above, leftovers (K % 32) added in double.  x has been rounded to f16 in the prologue (ggml.c:11141-11157).
__device__ __forceinline__ float dot_f16_row(const DevMat& w, int row, const uint8_t* smem, int lane) {
  const uint16_t* xa = (const uint16_t*)smem;
  const uint16_t* wr = (const uint16_t*)w.qs + (size_t)row * w.K;
  const int np = w.K & ~31;
  float s = 0.f;
  for (int i = lane; i < np; i += 32) s = __fmaf_rn(h2f(__ldg(wr + i)), h2f(xa[i]), s);
  double sumf = (double)warp_reduce_f32x8(s);
  for (int i = np; i < w.K; i++) sumf += (double)__fmul_rn(h2f(__ldg(wr + i)), h2f(xa[i]));
  return (float)sumf;
}
// F32 weights: ggml_vec_dot_f32 (ggml.c:2330-2365) has the same 4x8-lane shape.
__device__ __forceinline__ float dot_f32_row(const DevMat& w, int row, const uint8_t* smem, int lane) {
  const float* xa = (const float*)smem;
  const float* wr = (const float*)w.qs + (size_t)row * w.K;
  const int np = w.K & ~31;
  float s = 0.f;
  for (int i = lane; i < np; i += 32) s = __fmaf_rn(__ldg(wr + i), xa[i], s);
  float sumf = warp_reduce_f32x8(s);
  for (int i = np; i < w.K; i++) sumf = __fmaf_rn(__ldg(wr + i), xa[i], sumf);
  return sumf;
}

// The table entry as F16C widens it: a NaN keeps its sign and payload (h2f's conversion would give the canonical NaN).  The
// tables hold NaNs where the reference's activation of an out-of-range index is one, e.g. SiLU(-inf) = -inf / inf.
__device__ __forceinline__ float table_f16(const uint16_t* tab, float x) {
  const uint16_t h = __ldg(tab + f2h(x));
  return (h & 0x7fffu) > 0x7c00u ? __uint_as_float(((uint32_t)(h & 0x8000u) << 16) | 0x7f800000u | ((uint32_t)(h & 0x3ffu) << 13)) : h2f(h);
}

// The value an output element stores: the row's sum v with the segment's epilogue.  res / res2 point at this element's
// residuals (read by EPI_ADD / EPI_ADD2 only); they may have been written earlier in the same persistent kernel: L2-coherent loads.
__device__ __forceinline__ float epilogue(int epi, float v, const float* res, const float* res2, const MVParams& p) {
  if (epi == EPI_ADD) return __fadd_rn(v, __ldcg(res));
  if (epi == EPI_ADD2) return __fadd_rn(__fadd_rn(v, __ldcg(res)), __ldcg(res2));
  if (epi == EPI_GELU) return table_f16(p.gelu_tab, v);
  if (epi == EPI_SILU) return table_f16(p.silu_tab, v);
  return v;
}
__device__ __forceinline__ void store_epilogue(const MVSeg& sg, const MVParams& p, int row, float v) { sg.out[row] = epilogue(sg.epi, v, sg.res + row, sg.res2 + row, p); }

// rows one warp task covers for a (non-K-quant) weight type
__host__ __device__ inline int rows_per_unit(int type) { return (type == GT_F16 || type == GT_F32) ? 1 : MV_ROWS; }

// ---------------------------------------------------------------------------------------------
// Q4_0 / Q5_0 / Q8_0 / Q4_1 / Q5_1 / F16 / F32 weights.  Persistent: one CTA per SM, warp tasks strided over all warps of the grid.
static __global__ void __launch_bounds__(MV_THREADS, 1) k_matvec(const __grid_constant__ MVParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ double red[3 * MV_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_trigger();
  NormPre np;
  preload_norm(np, p);
  pdl_wait();   // everything above touched only weights and shared memory; the input vector is the predecessor's output
  stage_activation<MV_THREADS, 0>(p, np, p.act, smem, red, blockIdx.x == 0);
  const ActView a = act_view(p.act, p.K, smem);
  const int gw = blockIdx.x * MV_WARPS + warp, nw = gridDim.x * MV_WARPS;
  int first = gw;   // global striding continues across segments so all warps stay busy
  for (int s = 0; s < p.nseg; s++) {
    const MVSeg& sg = p.seg[s];
    const int type = sg.w.type;
    const int rpu = rows_per_unit(type);
    const int units = (sg.w.M + rpu - 1) / rpu;
    int un = first;
    for (; un < units; un += nw) {
      if (rpu == 1) {
        const float v = type == GT_F16 ? dot_f16_row(sg.w, un, smem, lane) : dot_f32_row(sg.w, un, smem, lane);
        if (lane == 0) store_epilogue(sg, p, un, v);
      } else {
        const int row = un * MV_ROWS + (lane >> 3);
        const float v = dot_legacy(sg.w, min(row, sg.w.M - 1), a, lane & 7);
        if ((lane & 7) == 0 && row < sg.w.M) store_epilogue(sg, p, row, v);
      }
    }
    first = un - units;   // where this warp lands in the next segment
  }
}

// host-side launch geometry shared by the engine and the op-level entry points
struct MVLaunch { int grid; size_t smem; };
inline MVLaunch matvec_launch_shape(const MVParams& p, int n_sm) {
  MVLaunch L;
  long units = 0;
  for (int s = 0; s < p.nseg; s++) { const int r = rows_per_unit(p.seg[s].w.type); units += (p.seg[s].w.M + r - 1) / r; }
  L.grid = (int)std::max<long>(1, std::min<long>((units + MV_WARPS - 1) / MV_WARPS, (long)n_sm));
  L.smem = (act_smem_bytes(p.act, p.K) + 15) & ~(size_t)15;
  return L;
}
constexpr int MV_SMEM_LIMIT = 200 * 1024;

// static: each translation unit launches / configures ITS OWN instantiation of the (static) kernel
static inline cudaError_t launch_matvec_kernel(const MVLaunch& L, cudaStream_t st, const MVParams& p, bool pdl = false) {
  return launch_kernel(k_matvec, dim3(L.grid), dim3(MV_THREADS), L.smem, st, pdl, p);
}
static inline cudaError_t matvec_set_smem_limit(int bytes) {
  return cudaFuncSetAttribute(k_matvec, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

}  // namespace ctb
