// Move-only owners of the library's CUDA resources: device and pinned host memory, streams, events, graphs and graph execs.
// Every handle, optional part and workspace holds its resources in these, so destroying or reassigning it frees them all,
// members in reverse declaration order.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <utility>

void lio_set_last_error(const char *file, int line, const char *msg);

namespace lio {

// Resources held by owners across the process (lio_live_resources).
extern std::atomic<long long> g_live_resources;

// One resource, released by D{}(h) when the owner is destroyed or assigned.  Converts to the raw handle, so kernel launches,
// parameter structs and CUDA calls take an owner where they take the handle.
template <class H, class D> class Own {
 public:
  Own() = default;
  Own(const Own &) = delete;
  Own &operator=(const Own &) = delete;
  Own(Own &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  template <class U> Own(Own<U, D> &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  Own &operator=(Own &&o) noexcept {
    if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); }
    return *this;
  }
  ~Own() { reset(); }
  operator H() const { return h_; }
  H get() const { return h_; }
  H operator->() const { return h_; }
  void reset() {
    if (h_) { D{}(h_); g_live_resources.fetch_sub(1, std::memory_order_relaxed); h_ = nullptr; }
  }
  // Takes h, just created by a call that returned e; on failure keeps the current resource and sets lio_last_error.
  bool take(cudaError_t e, H h, const char *what) {
    if (e != cudaSuccess) { lio_set_last_error(__FILE__, __LINE__, what ? what : cudaGetErrorString(e)); return false; }
    reset();
    h_ = h;
    if (h_) g_live_resources.fetch_add(1, std::memory_order_relaxed);
    return true;
  }

 private:
  template <class, class> friend class Own;
  H h_ = nullptr;
};

struct FreeDev { void operator()(void *p) const { cudaFree(p); } };
struct FreeHost { void operator()(void *p) const { cudaFreeHost(p); } };
struct DestroyStream { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct DestroyEvent { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct DestroyGraph { void operator()(cudaGraph_t g) const { cudaGraphDestroy(g); } };
struct DestroyGraphExec { void operator()(cudaGraphExec_t x) const { cudaGraphExecDestroy(x); } };

template <class T> using DevMem = Own<T *, FreeDev>;
template <class T> using HostMem = Own<T *, FreeHost>;   // cudaMallocHost and cudaHostAlloc (mapped) memory
using Stream = Own<cudaStream_t, DestroyStream>;
using Event = Own<cudaEvent_t, DestroyEvent>;
using Graph = Own<cudaGraph_t, DestroyGraph>;
using GraphExec = Own<cudaGraphExec_t, DestroyGraphExec>;

// The creation helpers allocate first and replace the owner's resource only on success: the old one stays on failure.
// They return false and set lio_last_error when the CUDA call fails.  n == 0 allocates one element.
template <class T> bool alloc(DevMem<T> &p, size_t n) {
  void *q = nullptr;
  const cudaError_t e = cudaMalloc(&q, sizeof(T) * (n ? n : 1));
  return p.take(e, (T *)q, "cudaMalloc failed");
}
template <class T> bool alloc_host(HostMem<T> &p, size_t n, unsigned flags = cudaHostAllocDefault) {
  void *q = nullptr;
  const cudaError_t e = cudaHostAlloc(&q, sizeof(T) * (n ? n : 1), flags);
  return p.take(e, (T *)q, "cudaHostAlloc failed");
}
inline bool create(Stream &s, unsigned flags = cudaStreamNonBlocking) {
  cudaStream_t h = nullptr;
  const cudaError_t e = cudaStreamCreateWithFlags(&h, flags);
  return s.take(e, h, "cudaStreamCreate failed");
}
inline bool create(Event &ev, unsigned flags = cudaEventDisableTiming) {
  cudaEvent_t h = nullptr;
  const cudaError_t e = cudaEventCreateWithFlags(&h, flags);
  return ev.take(e, h, "cudaEventCreate failed");
}
// Ends the capture on s: g owns whatever graph it produced, also when the capture failed.  Returns the capture's result.
inline cudaError_t end_capture(cudaStream_t s, Graph &g) {
  cudaGraph_t h = nullptr;
  const cudaError_t e = cudaStreamEndCapture(s, &h);
  g.take(cudaSuccess, h, nullptr);
  return e;
}
inline bool instantiate(GraphExec &x, cudaGraph_t g) {
  cudaGraphExec_t h = nullptr;
  const cudaError_t e = cudaGraphInstantiate(&h, g, 0);
  return x.take(e, h, nullptr);
}

}  // namespace lio
