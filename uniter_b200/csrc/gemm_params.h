// Shared between the GEMM device code (gemm_impl.cuh) and its C entry point (gemm.cu).
#pragma once
#include <stdint.h>

namespace ub {

constexpr int BM = 128;   // accumulator rows per CTA (two consumer warpgroups of 64)
constexpr int BK = 64;    // 64 x 16-bit = one 128-byte swizzle row

struct GemmParams {
  int M, N, K;
  int epilogue;
  const void* bias;
  const void* residual;
  const void* aux;
  void* out;
  void* out2;
  float* colsum;
  long long ldr, ldaux, ldo;
  uint32_t drop_thr16;
  float drop_inv_keep;
  uint32_t seed_lo, seed_hi, stream_lo, stream_hi;
  const unsigned long long* rng_dev;   // optional device-side stream offset (graph replay)
  int tiles_m, tiles_n;
  int ksplit;          // >= 1: work unit = (tile, k-slice); > 1 needs the fp32 atomic epilogue
  int kb_per_split;    // k-blocks per slice
};


// Grouped launch: up to 4 independent problems with the same K, operand majors (MN, MN) and
// epilogue (the four weight-gradient GEMMs of one encoder layer) share one persistent grid.
constexpr int GEMM_MAX_GROUP = 4;
struct GroupedParams {
  int nprob, K, epilogue;
  int bn;                               // N tile of every problem: 128, 192 or 256
  int M[GEMM_MAX_GROUP], N[GEMM_MAX_GROUP];
  void* out[GEMM_MAX_GROUP];
  long long ldo[GEMM_MAX_GROUP];
  int tiles_n[GEMM_MAX_GROUP];
  int tile_start[GEMM_MAX_GROUP + 1];   // prefix sums of the per-problem tile counts
};

}  // namespace ub
