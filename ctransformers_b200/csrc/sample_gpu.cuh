// Device half of ctransformers_llm_sample (reference: llama_llm::Sample, models/llms/llama.cc:53-84): the repetition penalty
// (llama.cpp:4025-4055) and the top-k cut (llama.cpp:3832-3857) over the n_vocab logits that are still on the device, so that
// only the surviving candidates travel to the host, where top-p / temperature / softmax / the seeded draw run unchanged
// (sampler.hpp).  One CTA: exact radix select of the k-th largest (penalised) logit, then a gather of everything >= it.
// The host falls back to the full-logits path when the cut is ambiguous (equal logits among the candidates: std::partial_sort
// leaves their order unspecified, so only the reference's own sort over all candidates reproduces it), and when some penalised
// logit is NaN (the reference's comparator is then no strict weak order, and only its own sort reproduces what it does).
#pragma once
#include <algorithm>
#include <cstdint>
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

static __global__ void __launch_bounds__(SG_THREADS) k_sample_topk(const float* logits, int n, const int* last_tokens, int n_last, float penalty, int k,
                                                                   SampleGpuOut* out) {
  __shared__ int last[SG_MAX_LAST];
  __shared__ unsigned hist[256];
  __shared__ uint32_t prefix, mask;
  __shared__ int want, n_out, nan;
  for (int j = threadIdx.x; j < n_last; j += SG_THREADS) last[j] = last_tokens[j];
  if (threadIdx.x == 0) { prefix = 0u; mask = 0u; want = k; n_out = 0; nan = 0; }
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
static inline void sg_launch(const float* logits, int n, const int* d_last, int n_last, float penalty, int k, SampleGpuOut* out, cudaStream_t st) {
  k_sample_topk<<<1, SG_THREADS, 0, st>>>(logits, n, d_last, n_last, penalty, std::min(k, n), out);
}
// What the host sampler can use of a result: the candidates' count (copied to ids / logits), or -1 when the device cannot answer
// (a NaN among the penalised logits, or more candidates than were written).
inline int sg_take(const SampleGpuOut& o, int* ids, float* logits) {
  if (o.nan || o.count < 0 || o.count > SG_MAX_OUT) return -1;
  for (int i = 0; i < o.count; i++) { ids[i] = o.id[i]; logits[i] = o.logit[i]; }
  return o.count;
}

}  // namespace ctb
