// Device half of ctransformers_llm_sample (reference: llama_llm::Sample, models/llms/llama.cc:53-84): the repetition penalty
// (llama.cpp:4025-4055) and the top-k cut (llama.cpp:3832-3857) over the n_vocab logits that are still on the device, so that
// only the surviving candidates travel to the host, where top-p / temperature / softmax / the seeded draw run unchanged
// (sampler.hpp).  One CTA per row (one sequence's logits): exact radix select of the k-th largest (penalised) logit, then a
// gather of everything >= it.
// The host falls back to the full-logits path when the cut is ambiguous (equal logits among the candidates: std::partial_sort
// leaves their order unspecified, so only the reference's own sort over all candidates reproduces it), and when some penalised
// logit is NaN (the reference's comparator is then no strict weak order, and only its own sort reproduces what it does).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

namespace ctb {

constexpr int SG_THREADS = 1024;
constexpr int SG_MAX_LAST = 256;    // repetition window the kernel handles (reference default 64)
constexpr int SG_MAX_OUT = 256;     // candidates returned at most

// nan: some penalised logit was NaN.  count may exceed SG_MAX_OUT (then only SG_MAX_OUT candidates are written).
struct SampleGpuOut { int count; int nan; int pad[2]; int id[SG_MAX_OUT]; float logit[SG_MAX_OUT]; };

// order-preserving: larger float -> larger key.  -0.0 gets the key of +0.0, as the reference's comparator sees them equal: two
// zeros split by the k-th largest logit then both make the cut, the count exceeds k, and the host decides.
__device__ __forceinline__ uint32_t sg_key(float v) {
  uint32_t u = __float_as_uint(v);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float sg_penalised(const float* logits, int i, const int* last, int n_last, float penalty) {
  float v = __ldcg(logits + i);
  if (n_last > 0 && penalty != 1.0f) {
    bool hit = false;
    for (int j = 0; j < n_last; j++) hit |= last[j] == i;
    if (hit) v = v <= 0.f ? __fmul_rn(v, penalty) : __fdiv_rn(v, penalty);
  }
  return v;
}

// The rows of one launch.  CTA r reads logits + row[r] * stride (n logits: the rows of a [slots][n_vocab] buffer are read in
// place), penalises the ids of last_tokens[last_off[r] .. last_off[r + 1]) by penalty[r], cuts at the k[r]-th largest and writes
// out[r].  Every array but logits and out lives in one argument block (sg_put / sg_rows), so one copy uploads a launch.
struct SgRows {
  const float* logits;
  size_t stride;
  const int* row;
  const int* k;
  const float* penalty;
  const int* last_off;
  const int* last_tokens;
  SampleGpuOut* out;
};

static __global__ void __launch_bounds__(SG_THREADS) k_sample_topk(const SgRows a, int n) {
  __shared__ int last[SG_MAX_LAST];
  __shared__ unsigned hist[256];
  __shared__ uint32_t prefix, mask;
  __shared__ int want, n_out, nan;
  const int r = blockIdx.x;
  const float* logits = a.logits + (size_t)a.row[r] * a.stride;
  const int l0 = a.last_off[r], n_last = a.last_off[r + 1] - l0;
  const float penalty = a.penalty[r];
  SampleGpuOut* out = a.out + r;
  for (int j = threadIdx.x; j < n_last; j += SG_THREADS) last[j] = a.last_tokens[l0 + j];
  if (threadIdx.x == 0) { prefix = 0u; mask = 0u; want = a.k[r]; n_out = 0; nan = 0; }
  __syncthreads();
  // radix select, most significant byte first: after each pass `prefix` fixes one more byte of the k-th largest key
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int b = threadIdx.x; b < 256; b += SG_THREADS) hist[b] = 0u;
    __syncthreads();
    const uint32_t pf = prefix, mk = mask;
    for (int i = threadIdx.x; i < n; i += SG_THREADS) {
      const uint32_t key = sg_key(sg_penalised(logits, i, last, n_last, penalty));
      if ((key & mk) == pf) atomicAdd(&hist[(key >> shift) & 0xffu], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int need = want, b = 255;
      for (; b > 0; b--) {
        if ((int)hist[b] >= need) break;
        need -= (int)hist[b];
      }
      want = need;
      prefix = pf | ((uint32_t)b << shift);
      mask = mk | (0xffu << shift);
    }
    __syncthreads();
  }
  const uint32_t kth = prefix;
  for (int i = threadIdx.x; i < n; i += SG_THREADS) {
    const float v = sg_penalised(logits, i, last, n_last, penalty);
    if (v != v) nan = 1;
    if (sg_key(v) >= kth) {
      const int slot = atomicAdd(&n_out, 1);
      if (slot < SG_MAX_OUT) { out->id[slot] = i; out->logit[slot] = v; }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) { out->count = n_out; out->nan = nan; }
}

// Host side.  The inputs k_sample_topk takes: a window of at most SG_MAX_LAST tokens, and 1 <= k <= SG_MAX_OUT / 2 (so that a
// few equal logits at the threshold still fit).
inline bool sg_accepts(int n_last, int k) { return n_last <= SG_MAX_LAST && k >= 1 && k <= SG_MAX_OUT / 2; }
// The window length a row is launched with: n_last <= 0 is no window, as for the host sampler (sample_token).
inline int sg_window(int n_last) { return std::max(n_last, 0); }
// The argument block of a launch of R rows whose windows hold n_tokens ids in all, as ints: row[R], k[R], penalty[R] (float
// bits), last_off[R + 1], then the windows one after another.
inline size_t sg_block_ints(int R, int n_tokens) { return (size_t)4 * R + 1 + n_tokens; }
// Row r of the block (rows are put in order 0, 1, ..): logits row `row` of n, this window (sg_window(n_last) of its ids count
// towards n_tokens), penalty and k (capped at n).
inline void sg_put(int* blk, int R, int r, int row, const int* last, int n_last, float penalty, int k, int n) {
  n_last = sg_window(n_last);
  int* off = blk + 3 * R;
  if (r == 0) off[0] = 0;
  blk[r] = row;
  blk[R + r] = std::min(k, n);
  memcpy(blk + 2 * R + r, &penalty, 4);
  off[r + 1] = off[r] + n_last;
  std::copy(last, last + n_last, blk + 4 * R + 1 + off[r]);
}
// The launch arguments over a device copy of the block.
inline SgRows sg_rows(const int* d_blk, int R, const float* logits, size_t stride, SampleGpuOut* out) {
  return SgRows{logits, stride, d_blk, d_blk + R, (const float*)(d_blk + 2 * R), d_blk + 3 * R, d_blk + 4 * R + 1, out};
}
static inline void sg_launch(const SgRows& a, int R, int n, cudaStream_t st) { k_sample_topk<<<R, SG_THREADS, 0, st>>>(a, n); }
// What the host sampler can use of a result: the candidates' count (copied to ids / logits), or -1 when the device cannot answer
// (a NaN among the penalised logits, or more candidates than were written).
inline int sg_take(const SampleGpuOut& o, int* ids, float* logits) {
  if (o.nan || o.count < 0 || o.count > SG_MAX_OUT) return -1;
  for (int i = 0; i < o.count; i++) { ids[i] = o.id[i]; logits[i] = o.logit[i]; }
  return o.count;
}

}  // namespace ctb
