// Scoring of logits rows on the device: for row r of n_vocab logits l and a target id t = targets[r] (-1: none),
//
//   logprob[r] = (double)l[t] - m - log(S),   m = the row's largest float,   S = Σ_i exp((double)l[i] - m)
//   greedy[r]  = t is the row's greedy pick (block_argmax: the reference's top_k = 1 scan, id 0 when nothing exceeds -inf or
//                when l[0] is NaN)
//
// The reference defines no log-probability; this is the project's own definition, in float64 over the float32 rows.  Its parts:
//   * S is summed in a fixed order: thread j of RL_THREADS adds the terms of ids j, j + RL_THREADS, j + 2 RL_THREADS, ... in
//     ascending order, then the RL_THREADS partial sums are added pairwise, part[j] += part[j + s] for s = RL_THREADS / 2 .. 1.
//   * Rows that are not all finite:
//       - any NaN in the row: logprob NaN;
//       - else c > 0 entries are +inf: logprob -log(c) when l[t] is +inf, else -inf (the limit of the formula);
//       - else every entry is -inf: logprob NaN (no distribution);
//       - else -inf entries add nothing to S, and a target at -inf gets -inf.
//   * No target (t = -1): logprob 0 and greedy 0.
// greedy follows block_argmax whatever the row holds, NaN included.  Targets outside [-1, n_vocab) are refused by the caller.
#pragma once
#include <cuda_runtime.h>

#include "attention.cuh"

namespace ctb {

constexpr int RL_THREADS = 256;

// one CTA per row
static __global__ void __launch_bounds__(RL_THREADS) k_row_logprob(const float* rows, int n_vocab, const int* targets, double* logprob, int* greedy) {
  __shared__ float bv[RL_THREADS / 32];
  __shared__ int bi[RL_THREADS / 32];
  __shared__ double part[RL_THREADS];
  __shared__ float wmax[RL_THREADS / 32];
  __shared__ int n_nan, n_inf;
  const float* l = rows + (size_t)blockIdx.x * n_vocab;
  const int t = targets[blockIdx.x];
  if (threadIdx.x == 0) { n_nan = 0; n_inf = 0; }
  float best;
  int pick;
  block_argmax<RL_THREADS, 0, false>(l, n_vocab, bv, bi, best, pick);   // (its barrier also publishes n_nan / n_inf = 0)
  // the largest value that is not NaN, and the NaN / +inf counts
  float mx = -INFINITY;
  int nan_c = 0, inf_c = 0;
  for (int i = threadIdx.x; i < n_vocab; i += RL_THREADS) {
    const float v = l[i];
    if (v != v) nan_c++;
    else {
      mx = fmaxf(mx, v);
      inf_c += v == INFINITY ? 1 : 0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = mx;
  if (nan_c) atomicAdd(&n_nan, nan_c);
  if (inf_c) atomicAdd(&n_inf, inf_c);
  __syncthreads();
  float m = wmax[0];
  for (int w = 1; w < RL_THREADS / 32; w++) m = fmaxf(m, wmax[w]);
  double s = 0.0;
  if (m > -INFINITY && m < INFINITY)
    for (int i = threadIdx.x; i < n_vocab; i += RL_THREADS) s += exp((double)l[i] - (double)m);
  part[threadIdx.x] = s;
  __syncthreads();
  for (int h = RL_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double lp;
    if (t < 0) lp = 0.0;
    else if (n_nan) lp = __longlong_as_double(0x7ff8000000000000ll);
    else if (n_inf) lp = l[t] == INFINITY ? -log((double)n_inf) : -(double)INFINITY;
    else if (m == -INFINITY) lp = __longlong_as_double(0x7ff8000000000000ll);
    else lp = ((double)l[t] - (double)m) - log(part[0]);
    logprob[blockIdx.x] = lp;
    greedy[blockIdx.x] = t >= 0 && t == pick ? 1 : 0;
  }
}

static inline void rl_launch(const float* rows, int n_rows, int n_vocab, const int* d_targets, double* d_logprob, int* d_greedy, cudaStream_t st) {
  if (n_rows > 0) k_row_logprob<<<n_rows, RL_THREADS, 0, st>>>(rows, n_vocab, d_targets, d_logprob, d_greedy);
}

}  // namespace ctb
