// Device-side data layout of the quantized hot path (sm_90a).
//
// Weights are NOT kept in GGUF's array-of-blocks form.  At load time every 2-D weight is repacked,
// byte for byte (same total size, so the HBM roofline denominator is unchanged):
//   K-quants (Q3_K / Q4_K / Q5_K / Q6_K): the STREAM layout of stream.cuh — 16-row tiles, block-major, every (tile, block) a
//   contiguous 16-byte-aligned piece of 16 x {110,144,176,210} bytes that one cp.async.bulk moves into shared memory and whose
//   interior is ordered for conflict-free 16-byte shared-memory loads of the mma.sync operand fragments.
//   Other types: per-tensor planes so that every lane of a warp issues 16-byte-aligned, fully coalesced loads no
//   matter how odd the source block size is (Q4_0 = 18 B, Q8_0 = 34 B):
//
//   type   plane qs (per row)          plane qh (per row)   plane d (per row)
//   Q4_0   nb x 16 B nibbles           -                    nb x fp16
//   Q5_0   nb x 16 B nibbles           nb x 4 B fifth bits  nb x fp16
//   Q4_1   nb x 16 B nibbles           -                    nb x fp16      + plane mn: nb x fp16 mins
//   Q5_1   nb x 16 B nibbles           nb x 4 B fifth bits  nb x fp16      + plane mn: nb x fp16 mins
//   Q8_0   nb x 32 B int8              -                    nb x fp16
//   F16    K x 2 B                     -                    -
//   F32    K x 4 B                     -                    -
//
// Block contents are exactly the reference's (k_quants.h:76-117, ggml.c:888-925); only their placement
// changes.  Activations are quantized on the fly to the reference's Q8_K / Q8_0 / Q8_1 (bit-exact) into
// shared memory (struct ActView) and never touch HBM.
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <utility>

namespace ctb {

enum : int { GT_F32 = 0, GT_F16 = 1, GT_Q4_0 = 2, GT_Q4_1 = 3, GT_Q5_0 = 6, GT_Q5_1 = 7, GT_Q8_0 = 8, GT_Q3_K = 11, GT_Q4_K = 12, GT_Q5_K = 13, GT_Q6_K = 14 };

struct DevMat {
  int type = -1;
  int K = 0, M = 0;     // K: contiguous (input) dim, M: rows (output features)
  int nb = 0;           // quant blocks per row
  const uint8_t* qs = nullptr;
  const uint8_t* qh = nullptr;
  const uint16_t* mn = nullptr;  // Q4_1 / Q5_1: the min plane.  The step kernel's phase descriptors embed DevMats, and dropping
                                 // these 8 bytes moved its dynamic shared memory by 32 B, which cost 2.5 % decode speed (H100 80GB HBM3, 700 W)
  const uint16_t* d = nullptr;
  const uint8_t* st = nullptr;   // K-quants: the stream layout of stream.cuh (16-row tiles, block-major; qs/qh/d stay null)
  size_t bytes = 0;     // total bytes of all planes (= GGUF tensor bytes)
};

__host__ __device__ inline bool type_is_kquant(int t) { return t == GT_Q3_K || t == GT_Q4_K || t == GT_Q5_K || t == GT_Q6_K; }
// activation format each weight type is multiplied with (reference: type_traits vec_dot_type, ggml.c:1638-1808)
enum : int { ACT_Q8_K = 0, ACT_Q8_0 = 1, ACT_F16 = 2, ACT_F32 = 3, ACT_Q8_1 = 4 };
__host__ __device__ inline int act_format_for(int t) {
  if (type_is_kquant(t)) return ACT_Q8_K;
  if (t == GT_Q4_0 || t == GT_Q5_0 || t == GT_Q8_0) return ACT_Q8_0;
  if (t == GT_Q4_1 || t == GT_Q5_1) return ACT_Q8_1;
  if (t == GT_F16) return ACT_F16;
  return ACT_F32;
}

// fp16 bit pattern <-> float, IEEE RNE (same results as the F16C instructions of the AVX2 reference build)
__device__ __forceinline__ float h2f(uint16_t h) { return __half2float(__ushort_as_half(h)); }
__device__ __forceinline__ uint16_t f2h(float f) { return __half_as_ushort(__float2half_rn(f)); }

// Programmatic dependent launch (sm_90+): a kernel lets its successor's CTAs start early (they prefetch weights and set up
// while this one drains) and the successor blocks in pdl_wait() until the whole predecessor grid has finished and its
// writes are visible.  Both are no-ops for a kernel launched without the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// launch with the programmatic-serialization attribute when pdl is set (the kernel may then start while its predecessor drains),
// and in clusters of `cluster` CTAs along x when that is more than 1
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, unsigned cluster,
                                                Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  unsigned n = 0;
  if (pdl) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (cluster > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = cluster; at[n].val.clusterDim.y = 1; at[n++].val.clusterDim.z = 1;
  }
  cfg.attrs = at; cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
  return launch_kernel_cluster(kernel, grid, block, smem, st, pdl, 1u, std::forward<Args>(args)...);
}

// dynamic shared memory a kernel can opt in to on the current device: the per-block limit less its static shared memory
template <typename Kernel>
static inline size_t max_dyn_smem(Kernel kernel) {
  cudaFuncAttributes fa{};
  if (cudaFuncGetAttributes(&fa, kernel) != cudaSuccess) return 0;
  int dev = 0, optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return (size_t)optin > fa.sharedSizeBytes ? (size_t)optin - fa.sharedSizeBytes : 0;
}

// named barrier over the first NT threads of the CTA (BAR = 0 with NT = blockDim.x is __syncthreads)
template <int BAR, int NT>
__device__ __forceinline__ void bar_sync() { asm volatile("bar.sync %0, %1;" ::"n"(BAR), "n"(NT) : "memory"); }

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// head sizes the attention kernels take (attention.cuh): even, because RoPE rotates pairs; 32 .. 256, so that a lane's share
// of the f16 dot's SIMD part is 1 .. 8 elements
__host__ __device__ inline bool attn_head_dim_ok(int hd) { return hd >= 32 && hd <= 256 && hd % 2 == 0; }
// ... of which 64 and 128 run in the kernels' own inline paths (the others in separate instantiations, attention.cuh)
__host__ __device__ inline bool attn_fast_hd(int hd) { return hd == 64 || hd == 128; }

}  // namespace ctb
