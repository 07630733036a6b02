// Move-only owners of CUDA resources: each one frees what it holds when it goes out of scope or takes another resource, so a
// buffer, event, stream or graph lives exactly as long as the engine or the call that holds it, also when that call throws.
#pragma once
#include <cuda_runtime.h>

#include <stdexcept>
#include <string>
#include <utility>

namespace ctb {

inline void cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string("CUDA error: ") + cudaGetErrorString(e) + " (" + what + ")");
}

// One handle H, released with Del.
template <typename H, cudaError_t (*Del)(H)>
class Owned {
 public:
  Owned() = default;
  Owned(Owned&& o) noexcept : h_(o.h_) { o.h_ = H{}; }
  Owned& operator=(Owned&& o) noexcept {
    if (this != &o) { reset(); h_ = o.h_; o.h_ = H{}; }
    return *this;
  }
  ~Owned() { reset(); }
  operator H() const { return h_; }
  void reset() { if (h_) Del(h_); h_ = H{}; }

 protected:
  H h_{};
};

class Event : public Owned<cudaEvent_t, cudaEventDestroy> {
 public:
  Event() = default;
  explicit Event(unsigned flags) { cuda_check(cudaEventCreateWithFlags(&h_, flags), "cudaEventCreateWithFlags"); }
};

class GraphExec : public Owned<cudaGraphExec_t, cudaGraphExecDestroy> {
 public:
  GraphExec() = default;
  explicit GraphExec(cudaGraph_t g) { cuda_check(cudaGraphInstantiate(&h_, g, 0), "cudaGraphInstantiate"); }
};

// A stream it created (and synchronises before destroying it), or one it only uses (set_stream).
class Stream {
 public:
  Stream() = default;
  explicit Stream(unsigned flags) : own_(true) { cuda_check(cudaStreamCreateWithFlags(&s_, flags), "cudaStreamCreateWithFlags"); }
  Stream(Stream&& o) noexcept { *this = std::move(o); }
  Stream& operator=(Stream&& o) noexcept {
    if (this != &o) { reset(); s_ = o.s_; own_ = o.own_; o.s_ = nullptr; o.own_ = false; }
    return *this;
  }
  ~Stream() { reset(); }
  operator cudaStream_t() const { return s_; }
  void set_stream(cudaStream_t s) { reset(); s_ = s; }
  void reset() {
    if (own_ && s_) { cudaStreamSynchronize(s_); cudaStreamDestroy(s_); }
    s_ = nullptr; own_ = false;
  }

 private:
  cudaStream_t s_ = nullptr;
  bool own_ = false;
};

// Device memory (Pinned = false) or pinned host memory, `mapped` for host words the device writes.  grow(bytes) reallocates
// when the buffer is smaller; what it held does not survive that.
template <bool Pinned>
class Mem {
 public:
  Mem() = default;
  explicit Mem(size_t bytes, bool mapped = false) : mapped_(mapped) { grow(bytes ? bytes : 1); }   // (never a null buffer)
  Mem(Mem&& o) noexcept { *this = std::move(o); }
  Mem& operator=(Mem&& o) noexcept {
    if (this != &o) { reset(); p_ = o.p_; n_ = o.n_; mapped_ = o.mapped_; o.p_ = nullptr; o.n_ = 0; }
    return *this;
  }
  ~Mem() { reset(); }
  void* grow(size_t bytes) {
    if (bytes <= n_) return p_;
    reset();
    if (Pinned) cuda_check(cudaHostAlloc(&p_, bytes, mapped_ ? cudaHostAllocMapped : cudaHostAllocDefault), "cudaHostAlloc");
    else cuda_check(cudaMalloc(&p_, bytes), "cudaMalloc");
    n_ = bytes;
    return p_;
  }
  void reset() {
    if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_);
    p_ = nullptr; n_ = 0;
  }
  void* get() const { return p_; }
  template <typename T> T* as() const { return (T*)p_; }
  explicit operator bool() const { return p_ != nullptr; }

 private:
  void* p_ = nullptr;
  size_t n_ = 0;
  bool mapped_ = false;
};
using DevMem = Mem<false>;
using HostMem = Mem<true>;

// The pinned entries (cap of them, `ints` ints each) through which launch state reaches one device target: put() fills the next
// entry and copies its first n ints to the target on the stream.  The copy runs later, so an entry is reused only after the
// copy that read it has run: when the ring wraps, it first synchronises the stream.
class StateRing {
 public:
  StateRing() = default;
  StateRing(int* target, int ints, int cap) : h_((size_t)ints * cap * 4), d_(target), ints_(ints), cap_(cap) {}
  template <typename Fill>
  cudaError_t put(cudaStream_t s, int n, Fill&& fill) {
    if (next_ > 0 && next_ % cap_ == 0)
      if (const cudaError_t e = cudaStreamSynchronize(s)) return e;
    int* e = h_.as<int>() + (size_t)(next_++ % cap_) * ints_;
    fill(e);
    return cudaMemcpyAsync(d_, e, (size_t)n * 4, cudaMemcpyHostToDevice, s);
  }

 private:
  HostMem h_;
  int* d_ = nullptr;
  int ints_ = 0, cap_ = 1;
  long next_ = 0;
};

}  // namespace ctb
