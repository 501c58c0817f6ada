// Shared host/device helpers for the dqn_zoo_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <string>

#include "../../include/dqn_zoo_b200.h"

namespace dz {
constexpr int kNumSMs = 132;   // H100 SXM: grid sizes of the grid-stride and one-CTA-per-SM kernels
}  // namespace dz

namespace dz {

extern thread_local std::string g_last_error;
extern std::atomic<int64_t> g_launches;

inline int fail(int code, const char* fmt, const char* a = "", const char* b = "") {
  char buf[512];
  snprintf(buf, sizeof(buf), fmt, a, b);
  g_last_error = buf;
  return code;
}

#define DZ_CUDA_OK(expr)                                                                     \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) return dz::fail(DZ_ECUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

// Returns a failing status code (anything but DZ_OK) from the enclosing function.
#define DZ_TRY(expr) do { int _s = (expr); if (_s != DZ_OK) return _s; } while (0)

// Optional per-launch CUDA-event timing (dz_profile_begin/end): used by bench.py to time the
// dominant kernel on its own stream.  Off in every timed run.
extern bool g_profile;
void profile_mark(const char* name, void* stream, bool begin);
void profile_geometry(unsigned gx, unsigned gy, unsigned bx);   // launch geometry of the record opened by profile_mark

// Programmatic dependent launch (PDL).  Every kernel of this library begins with pdl_enter() = griddepcontrol.wait
// and is launched with the programmatic-stream-serialization attribute: the next kernel's launch and block
// scheduling overlap the tail of the previous one, and all of its global-memory traffic still comes after
// everything it depends on has completed and is visible.  Kernel-to-kernel edges captured into the CUDA graph become
// programmatic edges.  Measured before the H100 port on the ~30-kernel learner steps: dqn 228 -> 217 us, rainbow
// 353 -> 338 us.  Dependents are not triggered early (griddepcontrol.launch_dependents at kernel entry): that was slower
// there (dqn 265 us), because the early CTAs spin at their wait and take issue slots and SM space from the kernel that
// is still running.
// Debug timeline (dz_debug_timeline): when a buffer is installed, thread 0 of block 0 of EVERY kernel appends
// (globaltimer, gridDim.x << 32 | gridDim.y << 16 | blockDim.x) right after its griddepcontrol.wait, i.e. at the moment
// everything it depends on has completed.  Read back after a CUDA-graph replay this is the true timeline of the step
// (launch gaps included), which neither per-launch events (eager only) nor ncu (serialised) can show.  Each translation
// unit has its own copy of the pointer (no relocatable device code); TimelineRegistrar collects the setters.
static __device__ unsigned long long* g_timeline = nullptr;
__device__ __forceinline__ void timeline_stamp() {
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    unsigned long long* tl = g_timeline;
    if (tl != nullptr) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      const unsigned int idx = atomicAdd(reinterpret_cast<unsigned int*>(tl), 1u);
      if (idx < 4000u) {
        tl[2 + 2 * idx] = t;
        tl[3 + 2 * idx] = ((unsigned long long)gridDim.x << 32) | ((unsigned long long)gridDim.y << 16) | blockDim.x;
      }
    }
  }
}
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  timeline_stamp();
}
typedef int (*timeline_setter_t)(unsigned long long*);
void timeline_register(timeline_setter_t fn);      // dz_replay.cu
static int timeline_set_this_tu(unsigned long long* p) { return (int)cudaMemcpyToSymbol(g_timeline, &p, sizeof(p)); }
struct TimelineRegistrar { TimelineRegistrar() { timeline_register(timeline_set_this_tu); } };
static TimelineRegistrar g_timeline_registrar;

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Every kernel launch goes through this so bench.py can report `gpu_launches`.
#define DZ_LAUNCH_NAMED(name, kernel, grid, block, smem, stream, ...)                        \
  do {                                                                                       \
    if (dz::g_profile) { dz::profile_mark(name, stream, true); dim3 _g(grid), _b(block); dz::profile_geometry(_g.x, _g.y, _b.x); } \
    dz::launch_kernel(kernel, dim3(grid), dim3(block), (size_t)(smem), (cudaStream_t)(stream), __VA_ARGS__); \
    if (dz::g_profile) dz::profile_mark(name, stream, false);                                \
    dz::g_launches.fetch_add(1, std::memory_order_relaxed);                                  \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess) return dz::fail(DZ_ECUDA, "launch %s: %s", name, cudaGetErrorString(_e)); \
  } while (0)
#define DZ_LAUNCH(kernel, grid, block, smem, stream, ...) \
  DZ_LAUNCH_NAMED(#kernel, kernel, grid, block, smem, stream, __VA_ARGS__)

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
// Output extent of a valid (unpadded) convolution: n inputs, kernel k, stride s.
inline int conv_out(int n, int k, int s) { return (n - k) / s + 1; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace dz
