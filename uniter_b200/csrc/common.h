// Host-side shared helpers: error reporting across the C ABI, TMA descriptor encoding through
// the driver entry point (no link-time dependency on libcuda, so the library loads on a
// CPU-only box), device properties cache.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ub200.h"

namespace ub {

int set_error(int code, const char* fmt, ...);  // stores message, returns code
#define UB_CHECK_ARG(cond, ...)                                    \
  do {                                                             \
    if (!(cond)) return ::ub::set_error(UB200_EINVAL, __VA_ARGS__); \
  } while (0)
#define UB_CHECK_CUDA(expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return ::ub::set_error(UB200_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                             __FILE__, __LINE__);                                             \
  } while (0)

// Dropout threshold of every dropout site for drop probability p in (0, 1): an element is dropped iff
// its 16-bit Philox value is below thr16, and kept values are scaled by inv_keep.  thr16 is clamped to
// [1, 65535], so a forward and a backward that both derive it from the same p agree on the mask for
// every p > 0, however small (oracle/philox.py dropout_params is the host mirror).
struct DropoutThreshold {
  uint32_t thr16;
  float inv_keep;
};
inline DropoutThreshold dropout_threshold(float p) {
  uint32_t thr = static_cast<uint32_t>(p * 65536.0f + 0.5f);
  if (thr > 65535u) thr = 65535u;
  if (thr == 0u) thr = 1u;
  return {thr, 65536.0f / static_cast<float>(65536u - thr)};
}

int num_sms();  // SM count of the current device (cached)
int deterministic();  // ub200_set_deterministic: launches use fixed-order reductions, no float atomics

// out[n] += sum_m x[m, n] in a fixed order (rows m ≡ lane mod 256, then a fixed tree): the bits depend
// on the values and their row indices only, and appended zero rows leave them unchanged.
// rows_dev (optional, device): only rows < min(rows, *rows_dev) are summed (e.g. &cu_seqlens[batch]).
int launch_colsum_det(int dtype, const void* x, float* out, int rows, int N, long long ld,
                      cudaStream_t stream, const int* rows_dev = nullptr);

// cudaFuncSetAttribute is per DEVICE: one bit per device in a per-instantiation mask (a process that
// drives several GPUs configures each of them once).  Returns true the first time for this device.
inline bool first_use_on_device(unsigned long long& mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (mask & bit) return false;
  mask |= bit;
  return true;
}

// 2-D row-major tensor [rows, cols] of 16-bit elements with row pitch `ld` (elements);
// box = box_cols x box_rows, 128-byte swizzle, zero OOB fill.  Returns 0 / negative code.
int make_tma_2d(CUtensorMap* out, const void* base, int dtype, uint64_t rows, uint64_t cols,
                uint64_t ld, uint32_t box_rows, uint32_t box_cols);


// Launch accounting + optional per-launch CUDA-event timing (bench.py's roofline pass).
// Every kernel launch site constructs a ProfScope right before the <<<>>>; it always counts the
// launch, and when profiling is enabled brackets it with a cudaEvent pair tagged with the
// role set by the caller (g_prof_tag, e.g. "FFN1 forward GEMM").
extern thread_local int g_prof_tag;
struct ProfScope {
  explicit ProfScope(cudaStream_t s);
  ~ProfScope();
  cudaStream_t stream;
  int slot;
};
struct ProfTag {
  explicit ProfTag(int t) : prev(g_prof_tag) { g_prof_tag = t; }
  ~ProfTag() { g_prof_tag = prev; }
  int prev;
};


// Launch with programmatic dependent launch enabled (and an optional 1-D cluster).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, int cluster, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = 1;
  ++n;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace ub
