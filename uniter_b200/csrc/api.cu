// Library identity, error channel and TMA descriptor encoding for libub200.so.
#include <cudaTypedefs.h>
#include <stdarg.h>
#include <stdio.h>

#include "common.h"

namespace ub {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

static int g_sm_reserve = 0;

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  int n = cached[dev] - g_sm_reserve;
  n &= ~1;                 // 2-CTA clusters need an even count
  return n < 2 ? 2 : n;
}

int set_sm_reserve(int n) {
  const int prev = g_sm_reserve;
  g_sm_reserve = n < 0 ? 0 : n;
  return prev;
}

static int g_deterministic = 0;

int deterministic() { return g_deterministic; }

static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

// A training step encodes ~400 descriptors, almost all of them identical to the previous step's
// (the caching allocator hands back the same blocks; weights never move).  A descriptor is a pure
// function of (base, dtype, rows, cols, ld, box), so a small direct-mapped, thread-local cache
// turns the driver call into a 56-byte compare + 128-byte copy.
struct TmaKey {
  const void* base;
  uint64_t rows, cols, ld;
  uint32_t box_rows, box_cols;
  int32_t dtype, valid;
};
struct alignas(64) TmaSlot {
  CUtensorMap map;
  TmaKey key;
};
constexpr int TMA_CACHE_SLOTS = 2048;
static thread_local TmaSlot* g_tma_cache = nullptr;

static inline uint32_t tma_hash(const TmaKey& k) {
  uint64_t h = reinterpret_cast<uint64_t>(k.base) * 0x9E3779B97F4A7C15ull;
  h ^= (k.rows * 0xC2B2AE3D27D4EB4Full) ^ (k.cols << 17) ^ (k.ld << 29) ^
       (static_cast<uint64_t>(k.box_rows) << 41) ^ (static_cast<uint64_t>(k.box_cols) << 7) ^
       static_cast<uint64_t>(k.dtype);
  h ^= h >> 29;
  h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 32;
  return static_cast<uint32_t>(h) & (TMA_CACHE_SLOTS - 1);
}

int make_tma_2d(CUtensorMap* out, const void* base, int dtype, uint64_t rows, uint64_t cols,
                uint64_t ld, uint32_t box_rows, uint32_t box_cols) {
  auto enc = get_encode();
  if (enc == nullptr)
    return set_error(UB200_ECUDA, "cuTensorMapEncodeTiled driver entry point unavailable");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (ld * 2) % 16 != 0)
    return set_error(UB200_EINVAL, "TMA operand must be 16-byte aligned with pitch %% 8 == 0 "
                                   "(base=%p ld=%llu)", base, (unsigned long long)ld);
  if (g_tma_cache == nullptr) g_tma_cache = new TmaSlot[TMA_CACHE_SLOTS]();
  TmaKey key{base, rows, cols, ld, box_rows, box_cols, dtype, 1};
  TmaSlot& slot = g_tma_cache[tma_hash(key)];
  if (slot.key.valid && slot.key.base == base && slot.key.rows == rows && slot.key.cols == cols &&
      slot.key.ld == ld && slot.key.box_rows == box_rows && slot.key.box_cols == box_cols &&
      slot.key.dtype == dtype) {
    *out = slot.map;
    return 0;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out,
                   dtype == UB200_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                       : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                   2, const_cast<void*>(base), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(UB200_ECUDA, "cuTensorMapEncodeTiled failed with CUresult %d "
                                  "(rows=%llu cols=%llu ld=%llu box=%ux%u)", (int)r,
                     (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld,
                     box_rows, box_cols);
  slot.map = *out;
  slot.key = key;
  return 0;
}


thread_local int g_prof_tag = 0;
static bool g_prof_on = false;
static unsigned long long g_launches = 0;
struct ProfRec { int tag; cudaEvent_t e0, e1; };
static ProfRec g_recs[8192];
static int g_nrec = 0;

ProfScope::ProfScope(cudaStream_t s) : stream(s), slot(-1) {
  ++g_launches;
  if (g_prof_on && g_nrec < 8192) {
    slot = g_nrec++;
    ProfRec& r = g_recs[slot];
    r.tag = g_prof_tag;
    if (!r.e0) { cudaEventCreate(&r.e0); cudaEventCreate(&r.e1); }
    cudaEventRecord(r.e0, stream);
  }
}
ProfScope::~ProfScope() {
  if (slot >= 0) cudaEventRecord(g_recs[slot].e1, stream);
}

}  // namespace ub

extern "C" {

unsigned long long ub200_launch_count(void) { return ub::g_launches; }

int ub200_set_sm_reserve(int n) { return ub::set_sm_reserve(n); }

int ub200_set_deterministic(int on) {
  const int prev = ub::g_deterministic;
  ub::g_deterministic = on ? 1 : 0;
  return prev;
}

int ub200_deterministic(void) { return ub::g_deterministic; }

int ub200_profile_enable(int on) {
  ub::g_prof_on = on != 0;
  if (on) ub::g_nrec = 0;
  return 0;
}

// Synchronises the device, sums the recorded launch durations per tag (ms) and launch counts
// per tag into ms_out[ntags] / count_out[ntags]; clears the record list.
int ub200_profile_collect(float* ms_out, int* count_out, int ntags) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return ub::set_error(UB200_ECUDA, "profile_collect: %s", cudaGetErrorString(e));
  for (int i = 0; i < ntags; ++i) { ms_out[i] = 0.f; count_out[i] = 0; }
  for (int i = 0; i < ub::g_nrec; ++i) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ub::g_recs[i].e0, ub::g_recs[i].e1);
    const int t = ub::g_recs[i].tag;
    if (t >= 0 && t < ntags) { ms_out[t] += ms; count_out[t] += 1; }
  }
  ub::g_nrec = 0;
  return 0;
}


int ub200_version(void) { return 200; /* 0.2.0 */ }

const char* ub200_last_error_string(void) { return ub::g_err; }

int ub200_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return ub::set_error(UB200_ECUDA, "no CUDA device: %s", cudaGetErrorString(e));
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0)
    return ub::set_error(UB200_EUNSUPPORTED, "libub200 is built for sm_90a only; device is sm_%d%d",
                         major, minor);
  return 0;
}

}  // extern "C"
