// GGUF array-of-blocks → device planes (layout table in device_types.cuh).  Shared by the engine's model
// upload and the op-level entry points.
#pragma once
#include "device_types.cuh"

namespace ctb {

struct PlaneSizes { size_t qs, qh, d, mn; };

inline PlaneSizes plane_sizes(int type, int M, int nb, size_t raw_bytes) {
  const size_t nblk = (size_t)M * nb;
  switch (type) {
    case GT_Q4_0: return {nblk * 16, 0, nblk * 2, 0};
    case GT_Q4_1: return {nblk * 16, 0, nblk * 2, nblk * 2};
    case GT_Q5_0: return {nblk * 16, nblk * 4, nblk * 2, 0};
    case GT_Q5_1: return {nblk * 16, nblk * 4, nblk * 2, nblk * 2};
    case GT_Q8_0: return {nblk * 32, 0, nblk * 2, 0};
    default: return {raw_bytes, 0, 0, 0};
  }
}

// GGUF array-of-blocks → planes (device_types.cuh), 2 bytes per thread-iteration (non-K-quant types; K-quants: stream.cuh).
static __global__ void k_repack(int type, const uint16_t* __restrict__ raw, size_t n_u16, uint16_t* qs, uint16_t* qh, uint16_t* d, uint16_t* mn) {
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n_u16; idx += (size_t)gridDim.x * blockDim.x) {
    const uint16_t v = raw[idx];
    switch (type) {
      case GT_Q4_0: {
        const size_t blk = idx / 9; const int o = (int)(idx % 9);
        if (o == 0) d[blk] = v; else qs[blk * 8 + (o - 1)] = v;
      } break;
      case GT_Q5_0: {   // 22 B: d, qh[4], qs[16]   (ggml.c:902-908)
        const size_t blk = idx / 11; const int o = (int)(idx % 11);
        if (o == 0) d[blk] = v; else if (o < 3) qh[blk * 2 + (o - 1)] = v; else qs[blk * 8 + (o - 3)] = v;
      } break;
      case GT_Q4_1: {   // 20 B: d, m, qs[16]   (ggml.c:896-900)
        const size_t blk = idx / 10; const int o = (int)(idx % 10);
        if (o == 0) d[blk] = v; else if (o == 1) mn[blk] = v; else qs[blk * 8 + (o - 2)] = v;
      } break;
      case GT_Q5_1: {   // 24 B: d, m, qh[4], qs[16]   (ggml.c:912-917)
        const size_t blk = idx / 12; const int o = (int)(idx % 12);
        if (o == 0) d[blk] = v; else if (o == 1) mn[blk] = v; else if (o < 4) qh[blk * 2 + (o - 2)] = v; else qs[blk * 8 + (o - 4)] = v;
      } break;
      case GT_Q8_0: {
        const size_t blk = idx / 17; const int o = (int)(idx % 17);
        if (o == 0) d[blk] = v; else qs[blk * 16 + (o - 1)] = v;
      } break;
      default: qs[idx] = v;
    }
  }
}

}  // namespace ctb
