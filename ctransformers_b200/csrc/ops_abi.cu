// Op-level C entry points (include/ctransformers_b200.h, part 2): each mirrors one ggml operator of the hot
// path with plain host pointers, runs the SAME device code the engine runs (stream.cuh / matvec.cuh / attention.cuh), and
// copies the result back.  Used by the parity tests and usable by a maintainer who wants to swap one op.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <ctime>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ctransformers_b200.h"
#include "attention.cuh"
#include "cuda_owned.cuh"
#include "engine.cuh"
#include "matvec.cuh"
#include "prefill.cuh"
#include "repack.cuh"
#include "sample_gpu.cuh"
#include "sampler.hpp"
#include "score_gpu.cuh"
#include "stream.cuh"
#include "tables.hpp"

using namespace ctb;

namespace {

#define OPS_CUDA(expr)                                                                                     \
  do {                                                                                                     \
    cudaError_t e__ = (expr);                                                                              \
    if (e__ != cudaSuccess) throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(e__) + " (" #expr ")"); \
  } while (0)

struct OpsTables {
  uint16_t *silu = nullptr, *gelu = nullptr, *ex = nullptr;
};

// built once per process, like the engine's
OpsTables& tables() {
  static OpsTables t;
  if (!t.silu) {
    const HostTables h = host_tables();
    OPS_CUDA(cudaMalloc(&t.silu, 65536 * 2)); OPS_CUDA(cudaMalloc(&t.gelu, 65536 * 2)); OPS_CUDA(cudaMalloc(&t.ex, 65536 * 2));
    OPS_CUDA(cudaMemcpy(t.silu, h.silu.data(), 65536 * 2, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(t.gelu, h.gelu.data(), 65536 * 2, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(t.ex, h.ex.data(), 65536 * 2, cudaMemcpyHostToDevice));
  }
  return t;
}

size_t raw_row_bytes(int type, int K) {
  switch (type) {
    case GT_F32: return (size_t)K * 4; case GT_F16: return (size_t)K * 2;
    case GT_Q4_0: return (size_t)K / 32 * 18; case GT_Q5_0: return (size_t)K / 32 * 22; case GT_Q8_0: return (size_t)K / 32 * 34;
    case GT_Q4_1: return (size_t)K / 32 * 20; case GT_Q5_1: return (size_t)K / 32 * 24;
    case GT_Q3_K: return (size_t)K / 256 * 110;
    case GT_Q4_K: return (size_t)K / 256 * 144; case GT_Q5_K: return (size_t)K / 256 * 176; case GT_Q6_K: return (size_t)K / 256 * 210;
  }
  throw std::runtime_error("unsupported ggml type " + std::to_string(type));
}
int block_elems(int type) {
  if (type_is_kquant(type)) return 256;
  return (type == GT_Q4_0 || type == GT_Q5_0 || type == GT_Q8_0 || type == GT_Q4_1 || type == GT_Q5_1) ? 32 : 1;
}

// the matrix in the engine's device layout, its planes in buffers that `keep` owns
DevMat upload(std::vector<DevMem>& keep, int type, const void* blocks, int K, int M) {
  if (K % block_elems(type)) throw std::runtime_error("K is not a multiple of the block size");
  const size_t bytes = raw_row_bytes(type, K) * M;
  DevMem raw(bytes);
  OPS_CUDA(cudaMemcpy(raw.get(), blocks, bytes, cudaMemcpyHostToDevice));
  DevMat m;
  m.type = type; m.K = K; m.M = M; m.nb = K / block_elems(type); m.bytes = bytes;
  if (type_is_kquant(type)) {   // the stream layout of the step kernel
    const size_t sb = st_matrix_bytes(type, M, m.nb);
    keep.emplace_back(sb);
    uint16_t* st = keep.back().as<uint16_t>();
    k_repack_stream<<<(int)std::min<size_t>((sb / 2 + 255) / 256, 4096), 256>>>(type, raw.as<uint8_t>(), M, m.nb, st);
    OPS_CUDA(cudaDeviceSynchronize());
    m.st = (const uint8_t*)st;
    return m;
  }
  const PlaneSizes ps = plane_sizes(type, M, m.nb, bytes);
  uint16_t* pl[4] = {nullptr, nullptr, nullptr, nullptr};
  const size_t sz[4] = {ps.qs, ps.qh, ps.d, ps.mn};
  for (int i = 0; i < 4; i++)
    if (sz[i]) { keep.emplace_back(sz[i]); pl[i] = keep.back().as<uint16_t>(); }
  k_repack<<<(int)std::min<size_t>((bytes / 2 + 255) / 256, 4096), 256>>>(type, raw.as<uint16_t>(), bytes / 2, pl[0], pl[1], pl[2], pl[3]);
  OPS_CUDA(cudaDeviceSynchronize());
  m.qs = (const uint8_t*)pl[0]; m.qh = (const uint8_t*)pl[1]; m.d = pl[2]; m.mn = pl[3];
  return m;
}

// the step kernel's watchdog words of this translation unit (stream.cuh st_fail), in host-mapped memory, so that a launch that
// trapped still tells which wait timed out; set once per process, like the tables
const int* watchdog_words() {
  static int* words = nullptr;
  if (!words) {
    OPS_CUDA(cudaHostAlloc((void**)&words, 16, cudaHostAllocMapped));
    memset(words, 0, 16);
    int* d = nullptr;
    OPS_CUDA(cudaHostGetDevicePointer((void**)&d, words, 0));
    OPS_CUDA(st_set_debug_words(d));
  }
  return words;
}

int sm_count() {
  int n_sm = 132;
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0);
  return n_sm;
}

// grid-barrier words of the persistent kernels (k_step and k_pstep both leave them zeroed when they end)
unsigned* sync_words() {
  static unsigned* d_sync = nullptr;
  if (!d_sync) { OPS_CUDA(cudaMalloc((void**)&d_sync, 64)); OPS_CUDA(cudaMemset(d_sync, 0, 64)); }
  return d_sync;
}

// the step kernel's launch shape for a program, exactly as the engine chooses it (shared-memory limits set)
StepLaunch plan_phases(const std::vector<Phase>& phs) {
  StepLaunch L = step_launch_plan(phs.data(), (int)phs.size(), sm_count());
  if (L.n_slots < ST_W) throw std::runtime_error("rows too long for the step kernel's shared memory");
  OPS_CUDA(step_set_smem_limit(L.smem));
  step_pair_choose(L, phs.data(), (int)phs.size());
  return L;
}

// a program of phases through the persistent step kernel, exactly as the engine launches it; returns the launch it made
StepLaunch run_phases(std::vector<Phase> phs) {
  unsigned* d_sync = sync_words();
  const StepLaunch L = plan_phases(phs);
  const std::vector<int> hb = step_bounds(phs.data(), (int)phs.size(), L.grid);
  DevMem dbounds(hb.size() * 4);
  OPS_CUDA(cudaMemcpy(dbounds.get(), hb.data(), hb.size() * 4, cudaMemcpyHostToDevice));
  DevMem dprog((phs.size() + 1) * sizeof(Phase));
  OPS_CUDA(cudaMemcpy(dprog.get(), phs.data(), phs.size() * sizeof(Phase), cudaMemcpyHostToDevice));
  OPS_CUDA(launch_step(L, 0, dprog.as<Phase>(), dbounds.as<int>(), (int)phs.size(), d_sync));
  OPS_CUDA(cudaGetLastError());
  OPS_CUDA(cudaDeviceSynchronize());
  return L;
}

// which kernel ran a mat-vec: k_step (1) or k_matvec (0), and the CTAs per cluster of its launch
struct MatvecLaunch { int kernel, cluster; };

// a mat-vec routed as Engine::push_matvec routes it, run `repeat` times back to back: one step-kernel program of that many
// phases, or that many k_matvec launches
MatvecLaunch run_matvec(MVParams& p, int repeat = 1) {
  p.silu_tab = tables().silu;
  p.gelu_tab = tables().gelu;
  if (step_supports(p)) {
    const StepLaunch L = run_phases(std::vector<Phase>(repeat, matvec_phase(p)));
    return {1, step_paired(L, false) ? 2 : 1};
  }
  static bool attr = false;
  if (!attr) {
    OPS_CUDA(matvec_set_smem_limit(MV_SMEM_LIMIT));
    attr = true;
  }
  const MVLaunch L = matvec_launch_shape(p, sm_count());
  for (int r = 0; r < repeat; r++) OPS_CUDA(launch_matvec_kernel(L, 0, p));
  OPS_CUDA(cudaGetLastError());
  return {0, 1};
}

// standalone wrappers around the prologue pieces, so the activation quantizers can be checked bit-for-bit
__global__ void __launch_bounds__(MV_THREADS) k_stage_dump(const __grid_constant__ MVParams q, int act, uint8_t* dump) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ double red[3 * MV_WARPS];
  NormPre np;
  preload_norm(np, q);
  stage_activation<MV_THREADS, 0>(q, np, act, smem, red, true);
  const size_t n = act_smem_bytes(act, q.K);
  for (size_t i = threadIdx.x; i < n; i += MV_THREADS) dump[i] = smem[i];
}

// the x_mode = 1 input path of the prologue on its own: out[i] = gate_act[i] * up[i] (gate_act = silu_table(gate), from the epilogue)
__global__ void __launch_bounds__(MV_THREADS) k_gate_dump(const __grid_constant__ MVParams q, float* out) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ double red[3 * MV_WARPS];
  NormPre np;
  preload_norm(np, q);
  stage_activation<MV_THREADS, 0>(q, np, ACT_F32, smem, red, false);
  const float* f = (const float*)smem;
  for (int i = threadIdx.x; i < q.K; i += MV_THREADS) out[i] = f[i];
}

// RoPE in place of the fp32 rows of blockIdx.x = 0 .. n_head-1 at position pos, as the attention kernels rotate q and k before
// rounding them to f16; block = hd/2 threads, one pair each
__global__ void k_rope_dump(float* x, const float2* rope, int pos, int hd, int neox) {
  float* row = x + (size_t)blockIdx.x * hd;
  int i0, i1;
  float o0, o1;
  rope_head_pair(row, threadIdx.x, hd, neox, rope[(size_t)pos * (hd / 2) + threadIdx.x], i0, i1, o0, o1);
  row[i0] = o0; row[i1] = o1;
}

int guarded(const char* what, const std::function<void()>& fn) {
  try {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) throw std::runtime_error("no CUDA device available (no CPU fallback)");
    fn();
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ctransformers-b200: %s failed: %s\n", what, e.what());
    return -1;
  }
}

void stage_to_host(const float* x, const float* w, const float* b, float* y_norm, int mode, float eps, int K, int act, std::vector<uint8_t>& dump) {
  DevMem dx((size_t)K * 4), dw((size_t)K * 4), db((size_t)K * 4), dy((size_t)K * 4);
  OPS_CUDA(cudaMemcpy(dx.get(), x, (size_t)K * 4, cudaMemcpyHostToDevice));
  if (w) OPS_CUDA(cudaMemcpy(dw.get(), w, (size_t)K * 4, cudaMemcpyHostToDevice));
  if (b) OPS_CUDA(cudaMemcpy(db.get(), b, (size_t)K * 4, cudaMemcpyHostToDevice));
  const size_t n = act_smem_bytes(act, K);
  DevMem dd(n);
  if (n > 48 * 1024) OPS_CUDA(cudaFuncSetAttribute(k_stage_dump, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n));
  MVParams q{};
  q.x = dx.as<float>(); q.norm_w = w ? dw.as<float>() : nullptr; q.norm_b = b ? db.as<float>() : nullptr; q.norm_out = dy.as<float>();
  q.norm_mode = mode; q.eps = eps; q.K = K;
  k_stage_dump<<<1, MV_THREADS, n>>>(q, act, dd.as<uint8_t>());
  OPS_CUDA(cudaGetLastError());
  dump.resize(n);
  OPS_CUDA(cudaMemcpy(dump.data(), dd.get(), n, cudaMemcpyDeviceToHost));
  if (y_norm) OPS_CUDA(cudaMemcpy(y_norm, dy.get(), (size_t)K * 4, cudaMemcpyDeviceToHost));
}

// KV caches in the reference's layouts (K [pos][n_kv*hd], V transposed [n_kv*hd][v_ld]), positions [0, n_pos)  <->  the
// device layouts of attention.cuh for a context of n_ctx (k_row / k_perm, kv_ctx_pad / v_perm); unset device entries are 0
void kv_to_device(const uint16_t* kref, const uint16_t* vref, int v_ld, int n_pos, int n_kv, int hd, int n_ctx, std::vector<uint16_t>& kp,
                  std::vector<uint16_t>& vp) {
  const int cp = kv_ctx_pad(n_ctx);
  kp.assign((size_t)n_ctx * n_kv * k_stride(hd), 0);
  vp.assign((size_t)n_kv * hd * cp, 0);
  for (int t = 0; t < n_pos; t++)
    for (int kh = 0; kh < n_kv; kh++)
      for (int e = 0; e < hd; e++) kp[k_row(kh, t, n_ctx, hd) + k_perm(e, hd)] = kref[((size_t)t * n_kv + kh) * hd + e];
  for (int ch = 0; ch < n_kv * hd; ch++)
    for (int t = 0; t < n_pos; t++) vp[(size_t)ch * cp + v_perm(t)] = vref[(size_t)ch * v_ld + t];
}
void kv_from_device(const std::vector<uint16_t>& kp, const std::vector<uint16_t>& vp, int n_kv, int hd, int n_ctx, uint16_t* kref, uint16_t* vref) {
  const int cp = kv_ctx_pad(n_ctx);
  for (int t = 0; t < n_ctx; t++)
    for (int kh = 0; kh < n_kv; kh++)
      for (int e = 0; e < hd; e++) kref[((size_t)t * n_kv + kh) * hd + e] = kp[k_row(kh, t, n_ctx, hd) + k_perm(e, hd)];
  for (int ch = 0; ch < n_kv * hd; ch++)
    for (int t = 0; t < n_ctx; t++) vref[(size_t)ch * n_ctx + t] = vp[(size_t)ch * cp + v_perm(t)];
}

// k_argmax over n device logits, as Engine::after_eval launches it: {pick, logits equal to the picked one}
void argmax_on_device(const float* d_logits, int n, int* pick2) {
  DevMem dout(8);
  k_argmax<<<1, ARGMAX_THREADS>>>(d_logits, n, dout.as<int>());
  OPS_CUDA(cudaGetLastError());
  OPS_CUDA(cudaMemcpy(pick2, dout.get(), 8, cudaMemcpyDeviceToHost));
}

// k_sample_topk over rows rows[0 ..) of a [rows][n] device buffer in one launch, as Engine::multi_sample launches it: result i is
// row q = rows[i]'s, with its window last_tokens[last_off[q] .. last_off[q + 1]), penalty[q] and k[q]
std::vector<SampleGpuOut> topk_rows_on_device(const float* d_logits, int n, const std::vector<int>& rows, const int* last_off, const int* last_tokens,
                                              const float* penalty, const int* k) {
  const int R = (int)rows.size();
  std::vector<SampleGpuOut> o(R);
  if (R == 0) return o;
  int n_tok = 0;
  for (int q : rows) n_tok += sg_window(last_off[q + 1] - last_off[q]);
  std::vector<int> blk(sg_block_ints(R, n_tok));
  for (int r = 0; r < R; r++) {
    const int q = rows[r];
    sg_put(blk.data(), R, r, q, last_tokens + last_off[q], last_off[q + 1] - last_off[q], penalty[q], k[q], n);
  }
  DevMem dblk(blk.size() * 4), dout((size_t)R * sizeof(SampleGpuOut));
  OPS_CUDA(cudaMemcpy(dblk.get(), blk.data(), blk.size() * 4, cudaMemcpyHostToDevice));
  sg_launch(sg_rows(dblk.as<int>(), R, d_logits, (size_t)n, dout.as<SampleGpuOut>()), R, n, 0);
  OPS_CUDA(cudaGetLastError());
  OPS_CUDA(cudaMemcpy(o.data(), dout.get(), (size_t)R * sizeof(SampleGpuOut), cudaMemcpyDeviceToHost));
  return o;
}

// k_sample_topk over n device logits, as Engine::topk_candidates launches it: one row
SampleGpuOut topk_on_device(const float* d_logits, int n, const int* last, int n_last, float penalty, int k) {
  const int off[2] = {0, sg_window(n_last)};
  return topk_rows_on_device(d_logits, n, {0}, off, last, &penalty, &k)[0];
}

// n_rows rows of n logits each, with their windows last_off[0 .. n_rows] into last_tokens: checked, then uploaded
void check_rows(int n_rows, int n, const int* last_off, const int* last_tokens) {
  if (n_rows < 1 || n < 1) throw std::runtime_error("no rows, or rows of no logits");
  for (int r = 0; r < n_rows; r++)
    if (last_off[r] < 0 || last_off[r + 1] < last_off[r]) throw std::runtime_error("window offsets that are not ascending");
  if (last_off[n_rows] > last_off[0] && !last_tokens) throw std::runtime_error("no window tokens");
}

}  // namespace

extern "C" {

int ctb_mul_mat(int type, const void* w_blocks, const float* x, float* dst, int K, int M, int N) {
  return guarded("ctb_mul_mat", [&] {
    std::vector<DevMem> keep;
    const DevMat w = upload(keep, type, w_blocks, K, M);
    DevMem dx((size_t)K * N * 4), dy((size_t)M * N * 4);
    OPS_CUDA(cudaMemcpy(dx.get(), x, (size_t)K * N * 4, cudaMemcpyHostToDevice));
    for (int n = 0; n < N; n++) {
      MVParams p{};
      p.x = dx.as<float>() + (size_t)n * K; p.norm_mode = NORM_NONE; p.K = K; p.act = act_format_for(type); p.nseg = 1;
      p.seg[0].w = w; p.seg[0].out = dy.as<float>() + (size_t)n * M; p.seg[0].epi = EPI_STORE;
      run_matvec(p);
    }
    OPS_CUDA(cudaMemcpy(dst, dy.get(), (size_t)M * N * 4, cudaMemcpyDeviceToHost));
  });
}

int ctb_quantize_row_q8_K(const float* x, void* y, int k) {
  return guarded("ctb_quantize_row_q8_K", [&] {
    if (k % 256) throw std::runtime_error("k must be a multiple of 256");
    std::vector<uint8_t> dump;
    stage_to_host(x, nullptr, nullptr, nullptr, NORM_NONE, 0.f, k, ACT_Q8_K, dump);
    const int nb = k / 256;
    const size_t off = ((size_t)k + 15) & ~(size_t)15;
    const float* d = (const float*)(dump.data() + off);
    const int16_t* bs = (const int16_t*)(dump.data() + off + q8k_d_bytes(k));
    uint8_t* out = (uint8_t*)y;   // block_q8_K: float d; int8 qs[256]; int16 bsums[16]  (k_quants.h:121-125)
    for (int b = 0; b < nb; b++) {
      memcpy(out + (size_t)b * 292, d + b, 4);
      for (int e = 0; e < 256; e++) {   // undo the lane-major shared-memory order (matvec.cuh q8k_word_offset)
        const int wd = e >> 2, sb = wd >> 3, ln = wd & 7;
        out[(size_t)b * 292 + 4 + e] = dump[(size_t)((b * 2 + (sb >> 2)) * 8 + ln) * 16 + (sb & 3) * 4 + (e & 3)];
      }
      memcpy(out + (size_t)b * 292 + 260, bs + (size_t)b * 16, 32);
    }
  });
}

int ctb_quantize_row_q8_0(const float* x, void* y, int k) {
  return guarded("ctb_quantize_row_q8_0", [&] {
    if (k % 32) throw std::runtime_error("k must be a multiple of 32");
    std::vector<uint8_t> dump;
    stage_to_host(x, nullptr, nullptr, nullptr, NORM_NONE, 0.f, k, ACT_Q8_0, dump);
    const int nb = k / 32;
    const size_t off = ((size_t)k + 15) & ~(size_t)15;
    const float* d = (const float*)(dump.data() + off);
    uint8_t* out = (uint8_t*)y;   // block_q8_0: fp16 d; int8 qs[32]  (ggml.c:920-925)
    for (int b = 0; b < nb; b++) {
      const uint16_t h = __half_as_ushort(__float2half_rn(d[b]));   // d[b] is already fp16-representable
      memcpy(out + (size_t)b * 34, &h, 2);
      memcpy(out + (size_t)b * 34 + 2, dump.data() + (size_t)b * 32, 32);
    }
  });
}

int ctb_quantize_row_q8_1(const float* x, void* y, int k) {
  return guarded("ctb_quantize_row_q8_1", [&] {
    if (k % 32) throw std::runtime_error("k must be a multiple of 32");
    std::vector<uint8_t> dump;
    stage_to_host(x, nullptr, nullptr, nullptr, NORM_NONE, 0.f, k, ACT_Q8_1, dump);
    const size_t off = ((size_t)k + 15) & ~(size_t)15;
    uint8_t* out = (uint8_t*)y;   // block_q8_1: float d; float s; int8 qs[32]  (ggml.c:928-932)
    for (int b = 0; b < k / 32; b++) {
      memcpy(out + (size_t)b * 40, dump.data() + off + (size_t)b * 8, 8);
      memcpy(out + (size_t)b * 40 + 8, dump.data() + (size_t)b * 32, 32);
    }
  });
}

int ctb_norm(int mode, const float* x, const float* w, const float* b, float* y, int n, float eps) {
  return guarded("ctb_norm", [&] {
    std::vector<uint8_t> dump;
    stage_to_host(x, w, b, y, mode, eps, n, ACT_F32, dump);
  });
}

int ctb_norm_path(int path, int mode, const float* x, const float* w, const float* b, float* y, int n, float eps) {
  return guarded("ctb_norm_path", [&] {
    if (path < 0 || path > 1) throw std::runtime_error("unknown norm path " + std::to_string(path));
    if (mode != NORM_RMS && mode != NORM_LAYER) throw std::runtime_error("norm mode 1 or 2");
    if (path == 0) {
      std::vector<uint8_t> dump;
      stage_to_host(x, w, b, y, mode, eps, n, ACT_F32, dump);
      return;
    }
    if (n < 256 || n % 256) throw std::runtime_error("the step kernel takes n a positive multiple of 256");
    // one mat-vec phase of the step kernel over 16 all-zero Q4_K rows: what is checked is the normalised vector CTA 0 writes
    const std::vector<uint8_t> zeros(raw_row_bytes(GT_Q4_K, n) * 16, 0);
    std::vector<DevMem> keep;
    const DevMat wm = upload(keep, GT_Q4_K, zeros.data(), n, 16);
    DevMem dx((size_t)n * 4), dw((size_t)n * 4), db((size_t)n * 4), dy((size_t)n * 4), dout(16 * 4);
    OPS_CUDA(cudaMemcpy(dx.get(), x, (size_t)n * 4, cudaMemcpyHostToDevice));
    if (w) OPS_CUDA(cudaMemcpy(dw.get(), w, (size_t)n * 4, cudaMemcpyHostToDevice));
    if (b) OPS_CUDA(cudaMemcpy(db.get(), b, (size_t)n * 4, cudaMemcpyHostToDevice));
    MVParams p{};
    p.x = dx.as<float>(); p.norm_w = w ? dw.as<float>() : nullptr; p.norm_b = b && mode == NORM_LAYER ? db.as<float>() : nullptr;
    p.norm_out = dy.as<float>(); p.norm_mode = mode; p.eps = eps; p.K = n; p.act = ACT_Q8_K; p.nseg = 1;
    p.seg[0].w = wm; p.seg[0].out = dout.as<float>(); p.seg[0].epi = EPI_STORE;
    p.silu_tab = tables().silu; p.gelu_tab = tables().gelu;
    run_phases({matvec_phase(p)});
    OPS_CUDA(cudaMemcpy(y, dy.get(), (size_t)n * 4, cudaMemcpyDeviceToHost));
  });
}

int ctb_norm_path_cluster(int n) {
  int cluster = -1;
  const int rc = guarded("ctb_norm_path_cluster", [&] {
    if (n < 256 || n % 256) throw std::runtime_error("the step kernel takes n a positive multiple of 256");
    MVParams p{};
    p.K = n; p.act = ACT_Q8_K; p.nseg = 1; p.norm_mode = NORM_RMS;
    p.seg[0].w.type = GT_Q4_K; p.seg[0].w.K = n; p.seg[0].w.M = 16; p.seg[0].w.nb = n / 256;
    cluster = step_paired(plan_phases({matvec_phase(p)}), false) ? 2 : 1;
  });
  return rc == 0 ? cluster : rc;
}

int ctb_rope(float* x, int n_heads, int head_dim, int pos, int mode, float freq_base, float freq_scale) {
  return guarded("ctb_rope", [&] {
    const int half = head_dim / 2;
    const std::vector<float2> tab = rope_table(pos + 1, head_dim, head_dim, freq_base, freq_scale);
    const size_t nq = (size_t)n_heads * head_dim;
    DevMem dq(nq * 4), dtab(tab.size() * 8);
    OPS_CUDA(cudaMemcpy(dq.get(), x, nq * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dtab.get(), tab.data(), tab.size() * 8, cudaMemcpyHostToDevice));
    k_rope_dump<<<n_heads, half>>>(dq.as<float>(), dtab.as<float2>(), pos, head_dim, (mode & 2) ? 1 : 0);
    OPS_CUDA(cudaGetLastError());
    OPS_CUDA(cudaMemcpy(x, dq.get(), nq * 4, cudaMemcpyDeviceToHost));
  });
}

int ctb_attention(const float* q, const uint16_t* kcache, const uint16_t* vcache, float* out, int n_head, int n_kv, int head_dim, int T,
                  int n_total, float kq_scale) {
  return guarded("ctb_attention", [&] {
    if (!attn_head_dim_ok(head_dim)) throw std::runtime_error("head_dim must be even, from 32 to 256");
    if (n_total < T) n_total = T;
    const size_t nq = (size_t)n_head * head_dim;
    std::vector<uint16_t> kp, vp;
    kv_to_device(kcache, vcache, T, T, n_kv, head_dim, n_total, kp, vp);
    // the kernel fuses RoPE + KV store for the current position: feed it an identity rotation (cos 1, sin 0 is exact) and the
    // current position's k/v taken back out of the caller's caches (f16 -> f32 -> f16 round-trips exactly)
    const int pos = T - 1;
    std::vector<float> kcur((size_t)n_kv * head_dim), vcur((size_t)n_kv * head_dim);
    for (int kh = 0; kh < n_kv; kh++)
      for (int e = 0; e < head_dim; e++) {
        kcur[(size_t)kh * head_dim + e] = __half2float(__ushort_as_half(kcache[((size_t)pos * n_kv + kh) * head_dim + e]));
        vcur[(size_t)kh * head_dim + e] = __half2float(__ushort_as_half(vcache[((size_t)kh * head_dim + e) * T + pos]));
      }
    std::vector<float2> ident((size_t)n_total * (head_dim / 2), make_float2(1.f, 0.f));
    DevMem dq(nq * 4), dk(kp.size() * 2), dv(vp.size() * 2), dout(nq * 4), dst(16), dkc(kcur.size() * 4), dvc(vcur.size() * 4), dtab(ident.size() * 8);
    OPS_CUDA(cudaMemcpy(dq.get(), q, nq * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dk.get(), kp.data(), kp.size() * 2, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dv.get(), vp.data(), vp.size() * 2, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dkc.get(), kcur.data(), kcur.size() * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dvc.get(), vcur.data(), vcur.size() * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dtab.get(), ident.data(), ident.size() * 8, cudaMemcpyHostToDevice));
    const int st[4] = {0, pos, 0, n_total};
    OPS_CUDA(cudaMemcpy(dst.get(), st, 16, cudaMemcpyHostToDevice));
    AttnParams ap{};
    ap.q = dq.as<float>(); ap.k = dkc.as<float>(); ap.v = dvc.as<float>(); ap.kc = dk.as<uint16_t>(); ap.vc = dv.as<uint16_t>();
    ap.out = dout.as<float>(); ap.exp_tab = tables().ex; ap.rope = dtab.as<float2>(); ap.state = dst.as<int>(); ap.kq_scale = kq_scale;
    ap.n_head = n_head; ap.n_kv = n_kv; ap.hd = head_dim; ap.n_ctx = n_total; ap.q_stride = (int)nq; ap.kv_stride = n_kv * head_dim; ap.neox = 0;
    const size_t smem = attn_smem_bytes(n_total, head_dim);
    OPS_CUDA(cudaFuncSetAttribute(attn_kernel(head_dim), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 48 * 1024)));
    attn_kernel(head_dim)<<<dim3(n_head, 1, attn_groups(head_dim)), ATTN_THREADS, smem>>>(ap);
    OPS_CUDA(cudaGetLastError());
    OPS_CUDA(cudaMemcpy(out, dout.get(), nq * 4, cudaMemcpyDeviceToHost));
  });
}

int ctb_attention_path(int path, const float* q, const float* k_new, const float* v_new, uint16_t* kcache, uint16_t* vcache, float* out,
                       int n_head, int n_kv, int head_dim, int n_ctx, int pos0, int n_tok, const int* n_total, int rope_mode, float freq_base,
                       float kq_scale) {
  return guarded("ctb_attention_path", [&] {
    const int hd = head_dim;
    if (path < 0 || path > 3) throw std::runtime_error("unknown attention path " + std::to_string(path));
    if (!attn_head_dim_ok(hd)) throw std::runtime_error("head_dim must be even, from 32 to 256");
    if (n_head < 1 || n_kv < 1 || n_head % n_kv) throw std::runtime_error("n_head must be a multiple of n_kv");
    if (n_tok < 1 || pos0 < 0 || pos0 + n_tok > n_ctx) throw std::runtime_error("the tokens' positions must lie inside the context");
    for (int i = 0; i < n_tok; i++)
      if (n_total[i] <= pos0 + i || n_total[i] > n_ctx) throw std::runtime_error("n_total[i] must lie in [position + 1, n_ctx]");
    const size_t nq = (size_t)n_head * hd, nkv = (size_t)n_kv * hd;
    std::vector<uint16_t> kp, vp;
    kv_to_device(kcache, vcache, n_ctx, n_ctx, n_kv, hd, n_ctx, kp, vp);
    const std::vector<float2> tab = rope_table(n_ctx, hd, hd, freq_base, 1.0f);
    // device state per token {token, position, step, n_total}; the batched kernel reads PB_T rows + the valid-token count
    std::vector<int> st((size_t)std::max(n_tok, PB_T) * 4 + 4, 0);
    for (int i = 0; i < std::max(n_tok, PB_T); i++) {
      const int k = std::min(i, n_tok - 1);
      st[(size_t)i * 4 + 1] = pos0 + k; st[(size_t)i * 4 + 3] = n_total[k];
    }
    if (path == 3) st[(size_t)PB_T * 4] = n_tok;
    DevMem dq(nq * n_tok * 4), dk(nkv * n_tok * 4), dv(nkv * n_tok * 4), dkc(kp.size() * 2), dvc(vp.size() * 2), dout(nq * n_tok * 4),
        dtab(tab.size() * 8), dst(st.size() * 4);
    OPS_CUDA(cudaMemcpy(dq.get(), q, nq * n_tok * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dk.get(), k_new, nkv * n_tok * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dv.get(), v_new, nkv * n_tok * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dkc.get(), kp.data(), kp.size() * 2, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dvc.get(), vp.data(), vp.size() * 2, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dtab.get(), tab.data(), tab.size() * 8, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dst.get(), st.data(), st.size() * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemset(dout.get(), 0, nq * n_tok * 4));
    AttnParams ap{};
    ap.q = dq.as<float>(); ap.k = dk.as<float>(); ap.v = dv.as<float>(); ap.kc = dkc.as<uint16_t>(); ap.vc = dvc.as<uint16_t>();
    ap.out = dout.as<float>(); ap.exp_tab = tables().ex; ap.rope = dtab.as<float2>(); ap.state = dst.as<int>(); ap.kq_scale = kq_scale;
    ap.n_head = n_head; ap.n_kv = n_kv; ap.hd = hd; ap.n_ctx = n_ctx; ap.q_stride = (int)nq; ap.kv_stride = (int)nkv; ap.neox = (rope_mode & 2) ? 1 : 0;
    if (path == 3) {   // one k_pstep launch of the engine's KV + ATTN phases (prefill_batch), with the engine's launch shape
      if (n_tok > PB_T) throw std::runtime_error("the batched kernel takes at most 32 tokens");
      int n_slots = 0;
      size_t smem = 0;
      // (the engine's scratch also holds the widest activation; a model with these heads has n_embd >= n_head * hd)
      if (!pstep_shape(pb_work_bytes((int)nq, n_ctx, hd), n_slots, smem)) throw std::runtime_error("n_ctx too long for the batched kernel's attention scratch");
      PPhase ph{};
      ph.at = ap; ph.state = dst.as<int>();
      PPhase prog[2] = {ph, ph};
      prog[0].kind = PP_KV; prog[1].kind = PP_ATTN;
      DevMem dprog(sizeof(prog));
      OPS_CUDA(cudaMemcpy(dprog.get(), prog, sizeof(prog), cudaMemcpyHostToDevice));
      OPS_CUDA(pstep_set_smem_limit(smem));
      OPS_CUDA(launch_pstep(sm_count(), n_slots, smem, 0, dprog.as<PPhase>(), 2, sync_words()));
    } else {   // one launch per token, in order, like decode_one
      if (path == 1) {
        Phase ph{};
        ph.kind = PH_ATTN; ph.q6 = 1; ph.at = ap;
        const StepLaunch L = step_launch_plan(&ph, 1, sm_count());
        if (!st_attn_ring_ok(n_ctx, L.n_slots)) throw std::runtime_error("the step kernel's ring cannot carry K / V at this n_ctx");
      }
      const size_t smem = attn_smem_bytes(n_ctx, hd);
      if (path == 0) OPS_CUDA(cudaFuncSetAttribute(attn_kernel(hd), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 48 * 1024)));
      for (int i = 0; i < n_tok; i++) {
        AttnParams a = ap;
        a.q += (size_t)i * nq; a.k += (size_t)i * nkv; a.v += (size_t)i * nkv; a.out += (size_t)i * nq; a.state += (size_t)i * 4;
        if (path == 0) {
          attn_kernel(hd)<<<dim3(n_head, 1, attn_groups(hd)), ATTN_THREADS, smem>>>(a);
          OPS_CUDA(cudaGetLastError());
        } else {
          Phase ph{};
          ph.kind = PH_ATTN; ph.q6 = path == 1 ? 1 : 0; ph.at = a;
          run_phases({ph});
        }
      }
    }
    OPS_CUDA(cudaDeviceSynchronize());
    OPS_CUDA(cudaMemcpy(out, dout.get(), nq * n_tok * 4, cudaMemcpyDeviceToHost));
    OPS_CUDA(cudaMemcpy(kp.data(), dkc.get(), kp.size() * 2, cudaMemcpyDeviceToHost));
    OPS_CUDA(cudaMemcpy(vp.data(), dvc.get(), vp.size() * 2, cudaMemcpyDeviceToHost));
    kv_from_device(kp, vp, n_kv, hd, n_ctx, kcache, vcache);
  });
}

int ctb_prefill_mul_mat(int nseg, const int* types, const void* const* w_blocks, const int* rows, int K, int n_tok, const float* x,
                        const float* x2, int norm_mode, const float* norm_w, const float* norm_b, float eps, const int* epi,
                        const float* res, const float* res2, float* out, int n_ctx, int head_dim, int* n_slots) {
  return guarded("ctb_prefill_mul_mat", [&] {
    if (nseg < 1 || nseg > MV_MAX_SEG) throw std::runtime_error("1 to 3 segments");
    if (K < 256 || K % 256) throw std::runtime_error("K must be a positive multiple of 256");
    if (n_tok < 1) throw std::runtime_error("n_tok must be at least 1");
    if (norm_mode < NORM_NONE || norm_mode > NORM_LAYER || (x2 && norm_mode != NORM_NONE)) throw std::runtime_error("norm mode 0, 1 or 2, and 0 with x2");
    if ((norm_mode != NORM_NONE && !norm_w) || (norm_mode == NORM_LAYER && !norm_b)) throw std::runtime_error("RMSNorm needs norm_w, LayerNorm norm_w and norm_b");
    if (norm_mode == NORM_NONE) norm_w = nullptr;   // the prologue applies whatever weight and bias it is given: only the mode's own
    if (norm_mode != NORM_LAYER) norm_b = nullptr;
    if (!attn_head_dim_ok(head_dim)) throw std::runtime_error("head_dim must be even, from 32 to 256");
    if (n_ctx < 1) throw std::runtime_error("n_ctx must be at least 1");
    int off[MV_MAX_SEG + 1] = {0};
    for (int s = 0; s < nseg; s++) {
      if (!type_is_kquant(types[s])) throw std::runtime_error("the batched kernel takes K-quant weights only");
      if (rows[s] < 1) throw std::runtime_error("every segment needs at least one row");
      if (epi[s] < EPI_STORE || epi[s] > EPI_SILU) throw std::runtime_error("unknown epilogue");
      if ((epi[s] == EPI_ADD || epi[s] == EPI_ADD2) && !res) throw std::runtime_error("ADD / ADD2 need res");
      if (epi[s] == EPI_ADD2 && !res2) throw std::runtime_error("ADD2 needs res2");
      off[s + 1] = off[s] + rows[s];
    }
    const int W = off[nseg];
    int slots = 0;
    size_t smem = 0;
    if (!pstep_shape(pb_work_bytes(K, n_ctx, head_dim), slots, smem)) throw std::runtime_error("no batched prefill at this n_ctx: its attention scratch does not fit");
    std::vector<DevMem> keep;
    DevMat mats[MV_MAX_SEG];
    for (int s = 0; s < nseg; s++) mats[s] = upload(keep, types[s], w_blocks[s], K, rows[s]);
    // PB_T-row token buffers, reused by every launch like the engine's batched buffers (rows past a short batch keep the previous
    // launch's values), and the QUANT phase's qbuf zeroed like the engine's
    DevMem dx((size_t)PB_T * K * 4), dx2((size_t)PB_T * K * 4), dout((size_t)PB_T * W * 4), dres((size_t)PB_T * W * 4), dres2((size_t)PB_T * W * 4),
        dnw((size_t)K * 4), dnb((size_t)K * 4), dq(pb_qbuf_bytes(K)), dst((PB_T * 4 + 4) * 4);
    OPS_CUDA(cudaMemset(dq.get(), 0, pb_qbuf_bytes(K)));
    OPS_CUDA(cudaMemset(dout.get(), 0, (size_t)PB_T * W * 4));
    if (norm_w) OPS_CUDA(cudaMemcpy(dnw.get(), norm_w, (size_t)K * 4, cudaMemcpyHostToDevice));
    if (norm_b) OPS_CUDA(cudaMemcpy(dnb.get(), norm_b, (size_t)K * 4, cudaMemcpyHostToDevice));
    MVParams m{};
    m.x = dx.as<float>(); m.x2 = x2 ? dx2.as<float>() : nullptr; m.x_mode = x2 ? 1 : 0;
    m.norm_w = norm_w ? dnw.as<float>() : nullptr; m.norm_b = norm_b ? dnb.as<float>() : nullptr; m.norm_mode = norm_mode; m.eps = eps;
    m.K = K; m.act = ACT_Q8_K; m.nseg = nseg; m.silu_tab = tables().silu; m.gelu_tab = tables().gelu;
    for (int s = 0; s < nseg; s++) {
      m.seg[s].w = mats[s]; m.seg[s].out = dout.as<float>() + off[s]; m.seg[s].epi = epi[s];
      if (epi[s] == EPI_ADD || epi[s] == EPI_ADD2) m.seg[s].res = dres.as<float>() + off[s];
      if (epi[s] == EPI_ADD2) m.seg[s].res2 = dres2.as<float>() + off[s];
    }
    struct Rows { const float* p; int ld; };
    const Rows bufs[5] = {{dx.as<float>(), K}, {dx2.as<float>(), K}, {dout.as<float>(), W}, {dres.as<float>(), W}, {dres2.as<float>(), W}};
    auto bat = [&](const float* p, int& ld) -> float* {
      ld = 0;
      if (!p) return nullptr;
      for (const Rows& b : bufs)
        if (p >= b.p && p < b.p + (size_t)PB_T * b.ld) { ld = b.ld; return const_cast<float*>(p); }
      throw std::runtime_error("pointer outside the token buffers");
    };
    std::vector<PPhase> prog;
    pb_matvec_phases(m, dq.as<uint8_t>(), dst.as<int>(), bat, prog);
    DevMem dprog((prog.size() + 1) * sizeof(PPhase));
    OPS_CUDA(cudaMemcpy(dprog.get(), prog.data(), prog.size() * sizeof(PPhase), cudaMemcpyHostToDevice));
    OPS_CUDA(pstep_set_smem_limit(smem));
    // launches of at most PB_T tokens over the same program and buffers, as eval_list cuts a run of prompt tokens
    for (int b = 0; b < n_tok; b += PB_T) {
      const int n = std::min(PB_T, n_tok - b);
      std::vector<int> st(PB_T * 4 + 4, 0);
      for (int i = 0; i < PB_T; i++) {
        const int k = std::min(i, n - 1);
        st[i * 4 + 1] = b + k; st[i * 4 + 3] = b + k + 1;
      }
      st[PB_T * 4] = n;
      OPS_CUDA(cudaMemcpy(dst.get(), st.data(), st.size() * 4, cudaMemcpyHostToDevice));
      OPS_CUDA(cudaMemcpy(dx.get(), x + (size_t)b * K, (size_t)n * K * 4, cudaMemcpyHostToDevice));
      if (x2) OPS_CUDA(cudaMemcpy(dx2.get(), x2 + (size_t)b * K, (size_t)n * K * 4, cudaMemcpyHostToDevice));
      if (res) OPS_CUDA(cudaMemcpy(dres.get(), res + (size_t)b * W, (size_t)n * W * 4, cudaMemcpyHostToDevice));
      if (res2) OPS_CUDA(cudaMemcpy(dres2.get(), res2 + (size_t)b * W, (size_t)n * W * 4, cudaMemcpyHostToDevice));
      OPS_CUDA(launch_pstep(sm_count(), slots, smem, 0, dprog.as<PPhase>(), (int)prog.size(), sync_words(), pstep_q3(prog)));
      OPS_CUDA(cudaDeviceSynchronize());
      OPS_CUDA(cudaMemcpy(out + (size_t)b * W, dout.get(), (size_t)n * W * 4, cudaMemcpyDeviceToHost));
    }
    if (n_slots) *n_slots = slots;
  });
}

int ctb_decode_mul_mat(int nseg, const int* types, const void* const* w_blocks, const int* rows, int K, int n_tok, const float* x,
                       const float* x2, int norm_mode, const float* norm_w, const float* norm_b, float eps, const int* epi,
                       const float* res, const float* res2, float* out, float* norm_out, int repeat, int* launch) {
  return guarded("ctb_decode_mul_mat", [&] {
    if (nseg < 1 || nseg > MV_MAX_SEG) throw std::runtime_error("1 to 3 segments");
    if (K < 1) throw std::runtime_error("K must be positive");
    if (n_tok < 1) throw std::runtime_error("n_tok must be at least 1");
    if (repeat < 1 || repeat > 4) throw std::runtime_error("repeat must be 1 to 4");
    if (norm_mode < NORM_NONE || norm_mode > NORM_LAYER || (x2 && norm_mode != NORM_NONE)) throw std::runtime_error("norm mode 0, 1 or 2, and 0 with x2");
    if ((norm_mode != NORM_NONE && !norm_w) || (norm_mode == NORM_LAYER && !norm_b)) throw std::runtime_error("RMSNorm needs norm_w, LayerNorm norm_w and norm_b");
    if (norm_mode == NORM_NONE) norm_w = nullptr;
    if (norm_mode != NORM_LAYER) norm_b = nullptr;
    int off[MV_MAX_SEG + 1] = {0};
    for (int s = 0; s < nseg; s++) {
      if (act_format_for(types[s]) != act_format_for(types[0])) throw std::runtime_error("the segments of one phase share an activation format");
      if (rows[s] < 1) throw std::runtime_error("every segment needs at least one row");
      if (epi[s] < EPI_STORE || epi[s] > EPI_SILU) throw std::runtime_error("unknown epilogue");
      if ((epi[s] == EPI_ADD || epi[s] == EPI_ADD2) && !res) throw std::runtime_error("ADD / ADD2 need res");
      if (epi[s] == EPI_ADD2 && !res2) throw std::runtime_error("ADD2 needs res2");
      off[s + 1] = off[s] + rows[s];
    }
    const int W = off[nseg];
    std::vector<DevMem> keep;
    DevMat mats[MV_MAX_SEG];
    for (int s = 0; s < nseg; s++) mats[s] = upload(keep, types[s], w_blocks[s], K, rows[s]);
    // one buffer of each kind, reused by every token's launch like the engine's decode buffers
    DevMem dx((size_t)K * 4), dx2((size_t)K * 4), dnw((size_t)K * 4), dnb((size_t)K * 4), dnorm((size_t)K * 4), dout((size_t)W * 4),
        dres((size_t)W * 4), dres2((size_t)W * 4);
    OPS_CUDA(cudaMemset(dout.get(), 0xff, (size_t)W * 4));
    OPS_CUDA(cudaMemset(dnorm.get(), 0xff, (size_t)K * 4));
    if (norm_w) OPS_CUDA(cudaMemcpy(dnw.get(), norm_w, (size_t)K * 4, cudaMemcpyHostToDevice));
    if (norm_b) OPS_CUDA(cudaMemcpy(dnb.get(), norm_b, (size_t)K * 4, cudaMemcpyHostToDevice));
    MVParams p{};
    p.x = dx.as<float>(); p.x2 = x2 ? dx2.as<float>() : nullptr; p.x_mode = x2 ? 1 : 0;
    p.norm_w = norm_w ? dnw.as<float>() : nullptr; p.norm_b = norm_b ? dnb.as<float>() : nullptr; p.norm_out = norm_out ? dnorm.as<float>() : nullptr;
    p.norm_mode = norm_mode; p.eps = eps; p.K = K; p.act = act_format_for(types[0]); p.nseg = nseg;
    for (int s = 0; s < nseg; s++) {
      p.seg[s].w = mats[s]; p.seg[s].out = dout.as<float>() + off[s]; p.seg[s].epi = epi[s];
      if (epi[s] == EPI_ADD || epi[s] == EPI_ADD2) p.seg[s].res = dres.as<float>() + off[s];
      if (epi[s] == EPI_ADD2) p.seg[s].res2 = dres2.as<float>() + off[s];
    }
    MatvecLaunch ran{};
    for (int i = 0; i < n_tok; i++) {   // one launch per token, as decode steps come
      OPS_CUDA(cudaMemcpy(dx.get(), x + (size_t)i * K, (size_t)K * 4, cudaMemcpyHostToDevice));
      if (x2) OPS_CUDA(cudaMemcpy(dx2.get(), x2 + (size_t)i * K, (size_t)K * 4, cudaMemcpyHostToDevice));
      if (res) OPS_CUDA(cudaMemcpy(dres.get(), res + (size_t)i * W, (size_t)W * 4, cudaMemcpyHostToDevice));
      if (res2) OPS_CUDA(cudaMemcpy(dres2.get(), res2 + (size_t)i * W, (size_t)W * 4, cudaMemcpyHostToDevice));
      ran = run_matvec(p, repeat);
      OPS_CUDA(cudaDeviceSynchronize());
      OPS_CUDA(cudaMemcpy(out + (size_t)i * W, dout.get(), (size_t)W * 4, cudaMemcpyDeviceToHost));
      if (norm_out) OPS_CUDA(cudaMemcpy(norm_out + (size_t)i * K, dnorm.get(), (size_t)K * 4, cudaMemcpyDeviceToHost));
    }
    if (launch) { launch[0] = ran.kernel; launch[1] = ran.cluster; }
  });
}

int ctb_xchg_mul_mat(int world, int rank, int n_embd, int n_head, int n_head_kv, int n_ff, int n_vocab, int n_layers, const int* types,
                     const void* const* w_blocks, const float* attn, const float* res0, const float* norm_w, float eps, const float* const* peers,
                     unsigned xc_base, int steps, float* out, float* sum_out, unsigned* ll, unsigned* sync2, int* launch) {
  return guarded("ctb_xchg_mul_mat", [&] {
    // everything is checked before the first device allocation: a program whose peers' entries are not all written would
    // spin until the watchdog traps
    if (world < 2 || world > XC_MAX_WORLD || rank < 0 || rank >= world) throw std::runtime_error("world must be 2 to 8 and rank below world");
    if (n_layers < 1 || steps < 1) throw std::runtime_error("n_layers and steps must be at least 1");
    if (n_vocab < 1) throw std::runtime_error("the head needs at least one row");
    const TPShard sh = tp_shard(n_embd, n_head, n_head_kv, n_ff, rank, world);   // (throws on a shape it does not split)
    const int hd = n_embd / n_head, per_kv = n_head / n_head_kv;
    if (sh.head1 <= sh.head0 || sh.ff1 <= sh.ff0) throw std::runtime_error("more ranks than 256-element blocks to share out");
    if (sh.head0 % per_kv || sh.head1 % per_kv) throw std::runtime_error("a rank's query heads must cover whole KV groups");
    const int q0 = sh.head0 * hd, q1 = sh.head1 * hd, g0 = sh.kv0 * hd, g1 = sh.kv1 * hd, f0 = sh.ff0, f1 = sh.ff1;
    const int qw = q1 - q0, gw = g1 - g0, fw = f1 - f0;
    if (q0 % 256 || q1 % 256 || f0 % 256 || f1 % 256) throw std::runtime_error("a K range off the 256-element block boundaries");
    const int n_mats = 7 * n_layers - 2, n_xchg = 2 * n_layers;
    for (int i = 0; i < n_mats; i++) {
      if (!w_blocks[i]) throw std::runtime_error("matrix " + std::to_string(i) + " is missing");
      if (!type_is_kquant(types[i])) throw std::runtime_error("the exchange runs in the step kernel: K-quant matrices only (matrix " + std::to_string(i) + ")");
    }
    if (!attn || !res0 || !norm_w) throw std::runtime_error("attention inputs, first residual and norm weights are required");
    for (int k = 0; k < n_xchg; k++)
      for (int r = 0; r < world; r++)
        if (r != rank && !peers[(size_t)k * world + r]) throw std::runtime_error("peer vector of rank " + std::to_string(r) + " in exchange " + std::to_string(k) + " is missing");

    std::vector<DevMem> keep;
    // rows [r0, r1) of a full K-wide matrix (column-parallel), or the blocks [k0, k1) of each of its M rows (row-parallel), packed
    // by the gather the engine's upload_matrix uses
    auto rows_of = [&](int i, int K, int r0, int r1) {
      return upload(keep, types[i], (const uint8_t*)w_blocks[i] + (size_t)r0 * raw_row_bytes(types[i], K), K, r1 - r0);
    };
    auto k_range_of = [&](int i, int K, int M, int k0, int k1) {
      const std::vector<uint8_t> g = gather_k_range((const uint8_t*)w_blocks[i], M, raw_row_bytes(types[i], K), raw_row_bytes(types[i], k0),
                                                    raw_row_bytes(types[i], k1 - k0));
      return upload(keep, types[i], g.data(), k1 - k0, M);
    };
    // consumer outputs side by side: per layer C_up {silu(w1), w3}, then C_qkv {wq, wk, wv}, or the head after the last layer
    std::vector<size_t> out_off(n_xchg + 1, 0);
    for (int c = 0; c < n_xchg; c++) out_off[c + 1] = out_off[c] + (c % 2 == 0 ? 2 * (size_t)fw : (c == n_xchg - 1 ? (size_t)n_vocab : (size_t)qw + 2 * gw));
    const size_t n_out = out_off[n_xchg], region = (size_t)2 * world * n_embd;   // region: uint2 ll[2][world][n_embd]
    DevMem dattn((size_t)n_layers * qw * 4), dres0((size_t)n_embd * 4), dnorm((size_t)n_xchg * n_embd * 4), dsum((size_t)n_xchg * n_embd * 4),
        dout(n_out * 4), dprod((size_t)n_embd * 4), dll((size_t)n_layers * world * region * 8), dsync(64);
    OPS_CUDA(cudaMemcpy(dattn.get(), attn, (size_t)n_layers * qw * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dres0.get(), res0, (size_t)n_embd * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dnorm.get(), norm_w, (size_t)n_xchg * n_embd * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemset(dsum.get(), 0xff, (size_t)n_xchg * n_embd * 4));
    OPS_CUDA(cudaMemset(dout.get(), 0xff, n_out * 4));
    OPS_CUDA(cudaMemset(dll.get(), 0, (size_t)n_layers * world * region * 8));   // as the engine's regions start
    OPS_CUDA(cudaMemset(dsync.get(), 0, 64));
    OPS_CUDA(cudaMemcpy(dsync.as<unsigned>() + 2, &xc_base, 4, cudaMemcpyHostToDevice));
    // The engine's regions hold two exchanges, one per parity half; a peer overwrites its slots of exchange k with those of
    // k + 2 once this rank has consumed k.  One launch on one GPU cannot wait for that, so each layer's pair of exchanges gets
    // its own W regions, laid out and used as the engine's: [layer][region of rank R][parity][slot of rank r][n_embd].
    auto ll_of = [&](int layer, int R) { return dll.as<uint2>() + ((size_t)layer * world + R) * region; };
    float* sums = dsum.as<float>();
    float* outs = dout.as<float>();

    // the program, numbered as Engine::build_ops numbers a fused tensor-parallel Llama layer (fill_xc, push_xchg, take_input,
    // mark_exchange), without the attention phase: per layer P_wo, C_up, P_down, then C_qkv or, after the last layer, the head
    std::vector<Phase> phs;
    int n_x = 0;              // exchanges so far in the program
    float* x_sum_into = nullptr;
    auto fill_xc = [&](XchgParams& xc, int role) {
      xc.world = world; xc.rank = rank; xc.index = n_x; xc.n = n_embd; xc.role = role;
      for (int r = 0; r < world; r++) xc.ll[r] = ll_of(n_x / 2, r);
    };
    auto push = [&](MVParams& p) {
      p.silu_tab = tables().silu; p.gelu_tab = tables().gelu;
      phs.push_back(matvec_phase(p));
    };
    auto push_xchg = [&](float* buf) { fill_xc(phs.back().xc, 2); x_sum_into = buf; };
    auto take_input = [&](MVParams& p) {
      p.x = (const float*)ll_of(n_x / 2, rank); p.x_mode = 2; p.x_parts = world; p.x_stride = n_embd; p.sum_out = x_sum_into;
    };
    auto mark_exchange = [&] { fill_xc(phs.back().xc, 1); n_x++; x_sum_into = nullptr; };
    const float* res = dres0.as<float>();   // the residual rank 0's next producer adds
    for (int l = 0; l < n_layers; l++) {
      const int m = 7 * l;
      {  // P_wo: the attention output's K range of wo (+ residual on rank 0)
        MVParams p{};
        p.x = dattn.as<float>() + (size_t)l * qw; p.norm_mode = NORM_NONE; p.K = qw; p.nseg = 1;
        p.seg[0] = MVSeg{k_range_of(m, n_embd, n_embd, q0, q1), dprod.as<float>(), rank == 0 ? res : nullptr, nullptr, rank == 0 ? EPI_ADD : EPI_STORE};
        push(p);
        push_xchg(sums + (size_t)n_x * n_embd);
      }
      {  // C_up: RMSNorm of the summed vector into this rank's rows of w1 (SiLU) and w3
        MVParams p{};
        p.norm_w = dnorm.as<float>() + (size_t)n_x * n_embd; p.norm_mode = NORM_RMS; p.eps = eps; p.K = n_embd;
        take_input(p);
        float* o = outs + out_off[n_x];
        p.nseg = 2;
        p.seg[0] = MVSeg{rows_of(m + 1, n_embd, f0, f1), o, nullptr, nullptr, EPI_SILU};
        p.seg[1] = MVSeg{rows_of(m + 2, n_embd, f0, f1), o + fw, nullptr, nullptr, EPI_STORE};
        res = p.sum_out;
        push(p);
        mark_exchange();
      }
      {  // P_down: w2's K range on silu(gate) * up (+ C_up's sum on rank 0)
        const float* gate = outs + out_off[n_x - 1];
        MVParams p{};
        p.x = gate; p.x2 = gate + fw; p.x_mode = 1; p.norm_mode = NORM_NONE; p.K = fw; p.nseg = 1;
        p.seg[0] = MVSeg{k_range_of(m + 3, n_ff, n_embd, f0, f1), dprod.as<float>(), rank == 0 ? res : nullptr, nullptr, rank == 0 ? EPI_ADD : EPI_STORE};
        push(p);
        push_xchg(sums + (size_t)n_x * n_embd);
      }
      {  // C_qkv into this rank's wq / wk / wv rows, or the replicated head after the last layer
        MVParams p{};
        p.norm_w = dnorm.as<float>() + (size_t)n_x * n_embd; p.norm_mode = NORM_RMS; p.eps = eps; p.K = n_embd;
        take_input(p);
        float* o = outs + out_off[n_x];
        if (l < n_layers - 1) {
          p.nseg = 3;
          p.seg[0] = MVSeg{rows_of(m + 4, n_embd, q0, q1), o, nullptr, nullptr, EPI_STORE};
          p.seg[1] = MVSeg{rows_of(m + 5, n_embd, g0, g1), o + qw, nullptr, nullptr, EPI_STORE};
          p.seg[2] = MVSeg{rows_of(m + 6, n_embd, g0, g1), o + qw + gw, nullptr, nullptr, EPI_STORE};
        } else {
          p.nseg = 1;
          p.seg[0] = MVSeg{rows_of(m + 4, n_embd, 0, n_vocab), o, nullptr, nullptr, EPI_STORE};
        }
        res = p.sum_out;
        push(p);
        mark_exchange();
      }
    }

    const StepLaunch L = plan_phases(phs);   // (the exchange build is never paired, whatever the plan says about pairs)
    const std::vector<int> hb = step_bounds(phs.data(), (int)phs.size(), L.grid);
    DevMem dbounds(hb.size() * 4), dprog((phs.size() + 1) * sizeof(Phase));
    OPS_CUDA(cudaMemcpy(dbounds.get(), hb.data(), hb.size() * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dprog.get(), phs.data(), phs.size() * sizeof(Phase), cudaMemcpyHostToDevice));
    const int* wd = watchdog_words();
    std::vector<uint2> slot(n_embd);
    for (int s = 0; s < steps; s++) {
      // the peers' entries of this launch's exchanges, numbered as the kernel numbers them, in this rank's regions
      const unsigned base = xc_base + (unsigned)s * (unsigned)n_xchg;
      for (int k = 0; k < n_xchg; k++) {
        const unsigned e = xc_epoch(base, k);
        for (int r = 0; r < world; r++) {
          if (r == rank) continue;
          const float* v = peers[(size_t)k * world + r];
          for (int i = 0; i < n_embd; i++) {
            memcpy(&slot[i].x, v + i, 4);
            slot[i].y = e;
          }
          OPS_CUDA(cudaMemcpy(ll_of(k / 2, rank) + ((size_t)(e & 1u) * world + r) * n_embd, slot.data(), (size_t)n_embd * 8, cudaMemcpyHostToDevice));
        }
      }
      OPS_CUDA(launch_step(L, 0, dprog.as<Phase>(), dbounds.as<int>(), (int)phs.size(), dsync.as<unsigned>(), false, nullptr, true));
      OPS_CUDA(cudaGetLastError());
      if (cudaDeviceSynchronize() != cudaSuccess) {
        const int* w = wd;
        throw std::runtime_error(std::string("launch ") + std::to_string(s) + " failed: " + cudaGetErrorString(cudaGetLastError()) + "; watchdog: wait " +
                                 std::to_string(w[0]) + " (" + WAIT_TEXT[w[0] > 0 && w[0] < W_CODES ? w[0] : 0] + ") in CTA " + std::to_string(w[1]) +
                                 ", aux " + std::to_string(w[2]) + ", thread " + std::to_string(w[3]));
      }
    }
    OPS_CUDA(cudaMemcpy(out, dout.get(), n_out * 4, cudaMemcpyDeviceToHost));
    OPS_CUDA(cudaMemcpy(sum_out, dsum.get(), (size_t)n_xchg * n_embd * 4, cudaMemcpyDeviceToHost));
    OPS_CUDA(cudaMemcpy(ll, dll.get(), (size_t)n_layers * world * region * 8, cudaMemcpyDeviceToHost));
    OPS_CUDA(cudaMemcpy(sync2, dsync.as<unsigned>() + 2, 4, cudaMemcpyDeviceToHost));
    if (launch) {
      const StepKernel k = step_kernel(L, true);
      launch[0] = k == k_step<true, false, false> || k == k_step<true, false, true>;
      launch[1] = k == k_step<true, false, true> || k == k_step<false, false, true> || k == k_step<false, true, true>;
      launch[2] = step_paired(L, true) ? 2 : 1;
    }
  });
}

int ctb_ffn_gate(int type, const void* w1_blocks, const void* w3_blocks, const float* x, float* out, int K, int M) {
  return guarded("ctb_ffn_gate", [&] {
    std::vector<DevMem> keep;
    const DevMat w1 = upload(keep, type, w1_blocks, K, M), w3 = upload(keep, type, w3_blocks, K, M);
    DevMem dx((size_t)K * 4), dg((size_t)M * 4), du((size_t)M * 4), dy((size_t)M * 4);
    OPS_CUDA(cudaMemcpy(dx.get(), x, (size_t)K * 4, cudaMemcpyHostToDevice));
    // as the engine does it: gate and up rows in one launch, SiLU(gate)*up where the down projection stages its input
    MVParams p{};
    p.x = dx.as<float>(); p.norm_mode = NORM_NONE; p.K = K; p.act = act_format_for(type); p.nseg = 2;
    p.seg[0].w = w1; p.seg[0].out = dg.as<float>(); p.seg[0].epi = EPI_SILU; p.seg[1].w = w3; p.seg[1].out = du.as<float>();
    run_matvec(p);
    const size_t smem = (size_t)M * 4 + 64;
    OPS_CUDA(cudaFuncSetAttribute(k_gate_dump, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 48 * 1024)));
    MVParams q{};
    q.x = dg.as<float>(); q.x2 = du.as<float>(); q.x_mode = 1; q.norm_mode = NORM_NONE; q.K = M;
    k_gate_dump<<<1, MV_THREADS, smem>>>(q, dy.as<float>());
    OPS_CUDA(cudaGetLastError());
    OPS_CUDA(cudaMemcpy(out, dy.get(), (size_t)M * 4, cudaMemcpyDeviceToHost));
  });
}

// Host-side view of how a K-quant mat-vec phase is cut up (no GPU needed): the 16-row tile range of every CTA.
int ctb_matvec_partition(const int* types, const int* rows, int nseg, int K, int n_sm, int* first_tile, int* meta) {
  if (nseg < 1 || nseg > MV_MAX_SEG || K <= 0 || K % 256 != 0 || n_sm < 1) return -1;
  MVParams p{};
  p.K = K; p.nseg = nseg; p.act = ACT_Q8_K;
  for (int s = 0; s < nseg; s++) {
    if (!type_is_kquant(types[s]) || rows[s] < 1) return -1;
    p.seg[s].w.type = types[s]; p.seg[s].w.K = K; p.seg[s].w.M = rows[s]; p.seg[s].w.nb = K / 256;
  }
  TileSpace ts;
  ts.init(p);
  const int nb = K / 256;
  long max_items = 0;
  for (int c = 0; c <= n_sm; c++) first_tile[c] = ts.boundary(c, n_sm);
  for (int c = 0; c < n_sm; c++) {
    long items = 0;
    for (int tile = first_tile[c]; tile < first_tile[c + 1]; tile++) {
      int tl = tile;
      items += st_chunks(types[ts.locate(tl)], nb);
    }
    max_items = std::max(max_items, items);
  }
  meta[0] = n_sm; meta[1] = ST_SLOT; meta[2] = ST_MAXT; meta[3] = ts.ntiles; meta[4] = ST_W; meta[5] = ST_ROWS; meta[6] = (int)max_items;
  meta[7] = st_chunk_blocks(GT_Q4_K) | (st_chunk_blocks(GT_Q5_K) << 8) | (st_chunk_blocks(GT_Q6_K) << 16) | (st_chunk_blocks(GT_Q3_K) << 24);
  return 0;
}

// Host-side view of how the paired step kernel splits the staging of a K-wide input (no GPU needed): block0[r] = first Q8_K
// block of cluster rank r (block0[2] = the end); returns 1 when a program of such phases can run paired (step_pair_fits), else 0.
int ctb_stage_pair_split(int K, int* block0) {
  if (K <= 0 || K % 256 != 0) return -1;
  for (int r = 0; r < 3; r++) block0[r] = pair_block0(K / 256, r);
  Phase ph{};
  ph.kind = PH_MATVEC;
  ph.mv.K = K;
  return step_pair_fits(&ph, 1) ? 1 : 0;
}

int ctb_get_row(int type, const void* table_blocks, int K, int n_rows, int row, float* out) {
  return guarded("ctb_get_row", [&] {
    const size_t rb = raw_row_bytes(type, K);
    DevMem dt(rb * n_rows), dtok(4), dout((size_t)K * 4);
    OPS_CUDA(cudaMemcpy(dt.get(), table_blocks, rb * n_rows, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dtok.get(), &row, 4, cudaMemcpyHostToDevice));
    EmbedParams em{};
    em.table = dt.as<uint8_t>(); em.row_bytes = rb; em.tokens = dtok.as<int>(); em.out = dout.as<float>(); em.type = type; em.K = K; em.n_vocab = n_rows;
    k_embed<<<1, 256>>>(em);
    OPS_CUDA(cudaGetLastError());
    OPS_CUDA(cudaMemcpy(out, dout.get(), (size_t)K * 4, cudaMemcpyDeviceToHost));
  });
}

int ctb_argmax_path(int path, const float* logits, int n, int* out) {
  return guarded("ctb_argmax_path", [&] {
    if (path < 0 || path > 1) throw std::runtime_error("unknown argmax path " + std::to_string(path));
    if (n < 1) throw std::runtime_error("no logits");
    DevMem dlog((size_t)n * 4);
    OPS_CUDA(cudaMemcpy(dlog.get(), logits, (size_t)n * 4, cudaMemcpyHostToDevice));
    if (path == 0) {
      argmax_on_device(dlog.as<float>(), n, out);
      return;
    }
    // one PH_PICK phase of the step kernel on the decode state out[0..4], as the last phase of the engine's step program
    const int step = out[2];
    if (step < 0 || step >= (1 << 20)) throw std::runtime_error("step out of range");
    DevMem dstate(5 * 4), dtok((size_t)(step + 1) * 4);
    OPS_CUDA(cudaMemcpy(dstate.get(), out, 5 * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemset(dtok.get(), 0xff, (size_t)(step + 1) * 4));
    Phase ph{};
    ph.kind = PH_PICK;
    ph.pk.logits = dlog.as<float>(); ph.pk.state = dstate.as<int>(); ph.pk.out_tokens = dtok.as<int>(); ph.pk.n = n;
    run_phases({ph});
    OPS_CUDA(cudaMemcpy(out, dstate.get(), 5 * 4, cudaMemcpyDeviceToHost));
    OPS_CUDA(cudaMemcpy(out + 5, dtok.as<int>() + step, 4, cudaMemcpyDeviceToHost));
  });
}

int ctb_sample_topk(const float* logits, int n, const int* last_tokens, int n_last, float repetition_penalty, int k, int* ids, float* lg) {
  int count = -1;
  const int rc = guarded("ctb_sample_topk", [&] {
    if (n < 1 || !sg_accepts(n_last, k)) throw std::runtime_error("n < 1, or a window or k the device sampler does not take");
    DevMem dlog((size_t)n * 4);
    OPS_CUDA(cudaMemcpy(dlog.get(), logits, (size_t)n * 4, cudaMemcpyHostToDevice));
    const SampleGpuOut o = topk_on_device(dlog.as<float>(), n, last_tokens, n_last, repetition_penalty, k);
    if (o.nan) { count = -2; return; }
    count = o.count;
    for (int i = 0; i < std::min(o.count, SG_MAX_OUT); i++) { ids[i] = o.id[i]; lg[i] = o.logit[i]; }
  });
  return rc == 0 ? count : -1;
}

int ctb_sample_device(const float* logits, int n, const int* last_tokens, int n_last, int top_k, float top_p, float temperature,
                      float repetition_penalty, int seed, int* used_device) {
  int tok = -1;
  const int rc = guarded("ctb_sample_device", [&] {
    if (n < 1) throw std::runtime_error("no logits");
    if (seed < 0) seed = (int)time(nullptr);
    std::mt19937 rng((unsigned)seed);
    DevMem dlog((size_t)n * 4);
    OPS_CUDA(cudaMemcpy(dlog.get(), logits, (size_t)n * 4, cudaMemcpyHostToDevice));
    bool dev = false;
    tok = sample_lazy(
        n, last_tokens, n_last, top_k, top_p, temperature, repetition_penalty, rng, dev,
        [&] {
          int pk[2];
          argmax_on_device(dlog.as<float>(), n, pk);
          return pk[1] == 1 ? pk[0] : -1;   // the rule of Engine::greedy_pick
        },
        [&](const int* last, int nl, float pen, int k, int* i, float* l) {
          if (!sg_accepts(nl, k)) return -1;
          return sg_take(topk_on_device(dlog.as<float>(), n, last, nl, pen, k), i, l);
        },
        [&] { return std::vector<float>(logits, logits + n); });
    *used_device = dev ? 1 : 0;
  });
  return rc == 0 ? tok : -1;
}

int ctb_sample_topk_rows(const float* logits, int n_rows, int n, const int* last_off, const int* last_tokens, const float* repetition_penalty,
                         const int* k, int* count, int* ids, float* lg) {
  return guarded("ctb_sample_topk_rows", [&] {
    check_rows(n_rows, n, last_off, last_tokens);
    std::vector<int> rows;
    for (int r = 0; r < n_rows; r++) {
      count[r] = -1;
      if (sg_accepts(last_off[r + 1] - last_off[r], k[r])) rows.push_back(r);
    }
    DevMem dlog((size_t)n_rows * n * 4);
    OPS_CUDA(cudaMemcpy(dlog.get(), logits, (size_t)n_rows * n * 4, cudaMemcpyHostToDevice));
    const std::vector<SampleGpuOut> o = topk_rows_on_device(dlog.as<float>(), n, rows, last_off, last_tokens, repetition_penalty, k);
    for (size_t i = 0; i < rows.size(); i++) {
      const int r = rows[i];
      count[r] = o[i].nan ? -2 : o[i].count;
      for (int j = 0; !o[i].nan && j < std::min(o[i].count, SG_MAX_OUT); j++) {
        ids[(size_t)r * SG_MAX_OUT + j] = o[i].id[j];
        lg[(size_t)r * SG_MAX_OUT + j] = o[i].logit[j];
      }
    }
  });
}

int ctb_sample_device_rows(const float* logits, int n_rows, int n, const int* last_off, const int* last_tokens, const int* top_k, const float* top_p,
                           const float* temperature, const float* repetition_penalty, const int* seed, int* tokens, int* used_device) {
  return guarded("ctb_sample_device_rows", [&] {
    check_rows(n_rows, n, last_off, last_tokens);
    DevMem dlog((size_t)n_rows * n * 4);
    OPS_CUDA(cudaMemcpy(dlog.get(), logits, (size_t)n_rows * n * 4, cudaMemcpyHostToDevice));
    // the device half as ctb_multi_sample_many runs it: every row's pick, one top-k launch over the rows that need a cut
    std::vector<int> picks((size_t)2 * n_rows), rows, row_of(n_rows, -1);
    for (int r = 0; r < n_rows; r++) {
      argmax_on_device(dlog.as<float>() + (size_t)r * n, n, &picks[2 * r]);
      const int nl = last_off[r + 1] - last_off[r];
      if (sample_is_greedy(top_k[r], repetition_penalty[r], nl) || !sg_accepts(nl, top_k[r])) continue;
      row_of[r] = (int)rows.size();
      rows.push_back(r);
    }
    const std::vector<SampleGpuOut> o = topk_rows_on_device(dlog.as<float>(), n, rows, last_off, last_tokens, repetition_penalty, top_k);
    for (int r = 0; r < n_rows; r++) {
      std::mt19937 rng((unsigned)(seed[r] < 0 ? (int)time(nullptr) : seed[r]));
      const float* row = logits + (size_t)r * n;
      bool dev = false;
      tokens[r] = sample_lazy(
          n, last_tokens ? last_tokens + last_off[r] : nullptr, last_off[r + 1] - last_off[r], top_k[r], top_p[r], temperature[r], repetition_penalty[r],
          rng, dev, [&] { return picks[2 * r + 1] == 1 ? picks[2 * r] : -1; },
          [&](const int*, int, float, int, int* i, float* l) { return row_of[r] < 0 ? -1 : sg_take(o[row_of[r]], i, l); },
          [&] { return std::vector<float>(row, row + n); });
      used_device[r] = dev ? 1 : 0;
    }
  });
}

int ctb_row_logprob(const float* rows, int n_rows, int n_vocab, const int* targets, double* logprob, int* greedy) {
  return guarded("ctb_row_logprob", [&] {
    if (n_rows < 1 || n_vocab < 1) throw std::runtime_error("no rows");
    for (int r = 0; r < n_rows; r++)
      if (targets[r] < -1 || targets[r] >= n_vocab) throw std::runtime_error("target " + std::to_string(targets[r]) + " of row " + std::to_string(r) + " is out of range");
    DevMem drows((size_t)n_rows * n_vocab * 4), dt((size_t)n_rows * 4), dlp((size_t)n_rows * 8), dg((size_t)n_rows * 4);
    OPS_CUDA(cudaMemcpy(drows.get(), rows, (size_t)n_rows * n_vocab * 4, cudaMemcpyHostToDevice));
    OPS_CUDA(cudaMemcpy(dt.get(), targets, (size_t)n_rows * 4, cudaMemcpyHostToDevice));
    rl_launch(drows.as<float>(), n_rows, n_vocab, dt.as<int>(), dlp.as<double>(), dg.as<int>(), 0);
    OPS_CUDA(cudaGetLastError());
    OPS_CUDA(cudaMemcpy(logprob, dlp.get(), (size_t)n_rows * 8, cudaMemcpyDeviceToHost));
    OPS_CUDA(cudaMemcpy(greedy, dg.get(), (size_t)n_rows * 4, cudaMemcpyDeviceToHost));
  });
}

}  // extern "C"
