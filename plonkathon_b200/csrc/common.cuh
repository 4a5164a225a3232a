// Shared host-side plumbing for libplonk_b200.so: error handling, the per-device context.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "curve.cuh"
#include "field.cuh"
#include "modinv.cuh"

namespace pb200 {

struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define PB_CUDA(expr)                                                                          \
  do {                                                                                         \
    cudaError_t e__ = (expr);                                                                  \
    if (e__ != cudaSuccess) {                                                                  \
      char b__[512];                                                                           \
      snprintf(b__, sizeof b__, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__),       \
               __FILE__, __LINE__);                                                            \
      throw pb200::Error(b__);                                                                 \
    }                                                                                          \
  } while (0)

#define PB_CHECK(cond, msg)                                                                    \
  do {                                                                                         \
    if (!(cond)) {                                                                             \
      char b__[512];                                                                           \
      snprintf(b__, sizeof b__, "%s (%s:%d)", msg, __FILE__, __LINE__);                        \
      throw pb200::Error(b__);                                                                 \
    }                                                                                          \
  } while (0)

// owning device buffer
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() {}
  explicit DevBuf(size_t n) { alloc(n); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void alloc(size_t n) {
    release();
    if (n) PB_CUDA(cudaMalloc(&p, n));
    bytes = n;
  }
  void ensure(size_t n) { if (n > bytes) alloc(n); }
  void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct NttPlan;
struct Srs;
struct Comm;
struct ShardTables;

struct Context {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaStream_t aux_stream = nullptr;    // independent transforms that overlap the MSM tails on `stream`
  cudaEvent_t aux_ev[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaStream_t copy_stream = nullptr;   // host->device staging that overlaps compute on `stream`
  cudaEvent_t copy_done[4] = {nullptr, nullptr, nullptr, nullptr};
  // the device's highest stream priority: the MSM phases that hardly use the integer multiplier (sort, stitch, upper
  // reduction levels), so that their blocks are dispatched ahead of another context's bucket accumulation (msm.cu)
  cudaStream_t prio_stream = nullptr;
  cudaEvent_t join_ev = nullptr;        // orders `stream` and `prio_stream` (stream_join)
  int sm_count = 132;
  std::map<int, std::unique_ptr<NttPlan>> plans;  // key: log_n * 2 + inverse
  DevBuf scratch[10];                              // reusable temporaries
  DevBuf msm_aff[6];                               // batched-affine bucket accumulation (msm.cu)
  Comm* comm = nullptr;                            // multi-GPU: this rank's communicator (comm.cuh), or null
  DevBuf gather;                                   // receive buffer of the sharded transforms' allgather
  std::map<int, std::unique_ptr<ShardTables>> shard_tables;  // per (log_n, inverse): twiddles of the sharded NTT join
  uint64_t launches = 0;                           // kernels launched through this context
  // optional per-kernel timing (bench.py roofline): CUDA event pairs on the stream the phase runs on (default:
  // `stream`)
  bool timing = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> timed[4];  // 0: MSM bucket accumulate, 1: NTT passes
  void time_begin(int cat, cudaStream_t on = nullptr) {
    if (!timing) return;
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    cudaEventRecord(a, on ? on : stream);
    timed[cat].push_back({a, b});
  }
  void time_end(int cat, cudaStream_t on = nullptr) {
    if (!timing) return;
    cudaEventRecord(timed[cat].back().second, on ? on : stream);
  }
  Context();
  ~Context();
};

NttPlan* get_plan(Context* ctx, int log_n, bool inverse);

// counts a kernel launched on `ctx` and reports a launch error
inline void launched(Context* ctx) {
  ctx->launches++;
  PB_CUDA(cudaGetLastError());
}

// grid and block size of a launch with one thread per item: kernel<<<PB_GRID(n, t), ...>>>
#define PB_GRID(n, t) (unsigned)(((n) + (t)-1) / (t)), (t)

// a field element through the read-only data cache, as two 16-byte loads
__device__ __forceinline__ Fr ldg_fr(const Fr* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 a = __ldg(q), b = __ldg(q + 1);
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}

// `waiter` runs nothing enqueued after this call before everything enqueued on `producer` so far has finished
inline void stream_join(Context* ctx, cudaStream_t waiter, cudaStream_t producer) {
  PB_CUDA(cudaEventRecord(ctx->join_ev, producer));
  PB_CUDA(cudaStreamWaitEvent(waiter, ctx->join_ev, 0));
}

}  // namespace pb200
