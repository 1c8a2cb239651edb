// GEMM with the residual + LayerNorm epilogue fused in (north star: "residual+LayerNorm epilogues"):
//
//   s = dropout(A W^T + bias) + residual          (model/layer.py:112-113, :153-154)
//   y = LayerNorm(s) * gamma + beta               (:114, :155; eps 1e-12, biased variance, fp32 stats)
//
// One kernel replaces GEMM(+bias+dropout+residual) -> s to HBM -> ln_fwd_kernel (read s, write y):
// the row statistics need the whole row of N = H columns, which is wider than one CTA's accumulator
// (128 x 768 fp32 = 384 accumulator registers per consumer thread), so the row is split over a CLUSTER of 4 CTAs along N
// (H = 768: 4 x 192, H = 1024: 4 x 256) that exchange per-row (mean, M2) through distributed shared
// memory:
//
//   pass 1  (epilogue warps, coalesced 4-lanes-per-row mapping of gemm_impl.cuh)
//           v = acc + bias -> dropout -> + residual -> round to 16 bit -> store s (saved for the
//           backward) and accumulate (count, mean, M2) of the ROUNDED values per row (Chan's
//           parallel update: no E[x^2] - E[x]^2 cancellation);
//   merge   4 lanes of a row (shuffles) -> barrier.cluster -> the 4 CTAs of the row (ld.shared::cluster) -> mean, rstd;
//   pass 2  re-read the CTA's own s (L2-hot, written by the same thread), normalise, scale, shift,
//           store y.
//
// The mainloop is the pipeline of gemm_kernel (TMA producer warpgroup, two wgmma consumer
// warpgroups with register accumulators); one 128 x BN tile per CTA.  A consumer warp owns 16 rows
// x all BN columns of the tile, so a row's CTA-local statistics never leave the warp.
#include "common.h"
#include "gemm_impl.cuh"

namespace ub {

struct LnEpiParams {
  const void* gamma;   // [N] 16-bit
  const void* beta;    // [N] 16-bit
  void* y;             // [M, N] 16-bit, pitch ldy
  long long ldy;
  float inv_n;         // 1 / N
};

constexpr int LN_CLUSTER = 4;
constexpr float LN_FUSED_EPS = 1e-12f;

template <int BN>
struct GemmLnCfg {
  static constexpr int BAR_BYTES = 256;
  static constexpr int STAT_BYTES = BM * 2 * 4;                   // this CTA's (mean, M2) per row
  static constexpr int SMEM_BYTES = GemmCfg<BN>::STAGES * GemmCfg<BN>::STAGE_BYTES + BAR_BYTES +
                                    GemmCfg<BN>::EPI_STAGE_BYTES + STAT_BYTES + 1024;
};

// (na, ma, M2a) <- merge with (nb, mb, M2b)
__device__ __forceinline__ void chan_merge(float& na, float& ma, float& M2a, float nb, float mb, float M2b) {
  const float n = na + nb;
  const float d = mb - ma;
  const float f = nb / n;
  ma = fmaf(d, f, ma);
  M2a = M2a + M2b + d * d * na * f;
  na = n;
}

__device__ __forceinline__ float2 ld_dsmem_f2(uint32_t cluster_addr) {
  float2 v;
  asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(cluster_addr) : "memory");
  return v;
}

template <int BN, bool kBF16, bool kDrop>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_ln_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const GemmParams p, const LnEpiParams q) {
  using Cfg = GemmCfg<BN>;
  using T16 = typename Elem<kBF16>::T;
  constexpr int CHUNKS = BN / 32;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + Cfg::STAGES;
  float* epi_stage_base = reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + GemmLnCfg<BN>::BAR_BYTES);
  float* cstat = epi_stage_base + EPI_WARPS * 16 * EPI_PITCH;     // [128][2]  (mean, M2) over BN columns

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int num_kb = (p.K + BK - 1) / BK;
  const int m0 = static_cast<int>(blockIdx.x / LN_CLUSTER) * BM;
  const int n0 = static_cast<int>(rank) * BN;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    fence_barrier_init();
  }
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();

  const bool is_epi = warp >= 4;
  const int cw = is_epi ? warp - 4 : 0;          // consumer warp: tile rows [16 cw, 16 cw + 16)
  const int sub_r = lane >> 2;
  const int cg = (lane & 3) * 8;
  float* stage = epi_stage_base + cw * (16 * EPI_PITCH);
  const int row_base = m0 + 16 * cw;
  float acc[BN / 2];
  if (!is_epi) {
    setmaxnreg_producer();
    // ===================================================================== TMA producer
    if (warp == 0 && lane == 0) {
      int st = 0;
      uint32_t phase = 0;
      produce_tile<BN, false, false, 1>(smem, full_bar, empty_bar, &tmA, &tmB, m0, n0, 0, num_kb, st, phase, 0u);
    }
  } else {
    setmaxnreg_consumer();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int st = 0;
    uint32_t phase = 0;
    consume_tile<BN, false, false, kBF16, 1>(acc, smem, full_bar, empty_bar, num_kb, cw >> 2, st, phase, 0u);
    const DropoutRng rng = make_rng(p);
    float cnt[2], mean[2], M2[2];
#pragma unroll
    for (int it = 0; it < 2; ++it) { cnt[it] = 0.f; mean[it] = 0.f; M2[it] = 0.f; }
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      const int col = n0 + c * 32 + cg;
      const uint4 bias4 = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.bias) + col));
      uint4 side[2];
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        const int row = row_base + it * 8 + sub_r;
        side[it] = make_uint4(0, 0, 0, 0);
        if (row < p.M)
          side[it] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.residual) +
                                                          static_cast<long long>(row) * p.ldr + col));
      }
      __syncwarp();
      stage_block<BN>(acc, c, lane, stage);
      __syncwarp();
      float bias8[8];
      unpack8_<kBF16>(bias4, bias8);
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        const int rr = it * 8 + sub_r;
        const int row = row_base + rr;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = stage[rr * EPI_PITCH + cg + i] + bias8[i];
        if (kDrop) {
          const uint64_t e = static_cast<uint64_t>(row) * static_cast<uint64_t>(p.N) + col;
          const uint4 rnd = rng.draw8(e >> 3);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = (rand16_of(rnd, i) < rng.thr16) ? 0.f : v[i] * rng.inv_keep;
        }
        float t[8];
        unpack8_<kBF16>(side[it], t);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] += t[i];
        // the LayerNorm of the reference acts on the 16-bit sum: round first, then take statistics
        uint4 s16;
        s16.x = Elem<kBF16>::pack(v[0], v[1]); s16.y = Elem<kBF16>::pack(v[2], v[3]);
        s16.z = Elem<kBF16>::pack(v[4], v[5]); s16.w = Elem<kBF16>::pack(v[6], v[7]);
        if (row < p.M)
          *reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.out) + static_cast<long long>(row) * p.ldo + col) = s16;
        unpack8_<kBF16>(s16, v);
        float m8 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) m8 += v[i];
        m8 *= 0.125f;
        float q8 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) { const float d = v[i] - m8; q8 = fmaf(d, d, q8); }
        if (c == 0) { cnt[it] = 8.f; mean[it] = m8; M2[it] = q8; }
        else chan_merge(cnt[it], mean[it], M2[it], 8.f, m8, q8);
      }
    }
    // the 4 lanes of a row (equal counts)
#pragma unroll
    for (int it = 0; it < 2; ++it) {
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        const float mb = __shfl_xor_sync(0xffffffffu, mean[it], off);
        const float qb = __shfl_xor_sync(0xffffffffu, M2[it], off);
        chan_merge(cnt[it], mean[it], M2[it], cnt[it], mb, qb);
      }
      if ((lane & 3) == 0) {
        float* w = cstat + (16 * cw + it * 8 + sub_r) * 2;
        w[0] = mean[it];
        w[1] = M2[it];
      }
    }
  }
  // ---- every CTA of the cluster has published its per-row partial statistics
  __syncwarp();
  cluster_sync_all();
  if (is_epi) {
    float mu[2], rs[2];
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const uint32_t local = smem_u32(cstat + (16 * cw + it * 8 + sub_r) * 2);
      float n = 0.f, m = 0.f, s2 = 0.f;
#pragma unroll
      for (int r4 = 0; r4 < LN_CLUSTER; ++r4) {
        const float2 pr = ld_dsmem_f2(mapa_shared(local, static_cast<uint32_t>(r4)));
        if (r4 == 0) { n = static_cast<float>(BN); m = pr.x; s2 = pr.y; }
        else chan_merge(n, m, s2, static_cast<float>(BN), pr.x, pr.y);
      }
      mu[it] = m;
      rs[it] = rsqrtf(s2 * q.inv_n + LN_FUSED_EPS);
    }
    // ---- pass 2: y = (s - mean) * rstd * gamma + beta over this warp's rows
#pragma unroll 1
    for (int c = 0; c < CHUNKS; ++c) {
      const int col = n0 + c * 32 + cg;
      float g8[8], b8[8];
      unpack8_<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(q.gamma) + col)), g8);
      unpack8_<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(q.beta) + col)), b8);
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        const int row = row_base + it * 8 + sub_r;
        if (row >= p.M) continue;
        // own store of pass 1 (same thread, same address): a plain (coherent) load
        const uint4 s16 = *reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.out) +
                                                          static_cast<long long>(row) * p.ldo + col);
        float v[8];
        unpack8_<kBF16>(s16, v);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = (v[i] - mu[it]) * rs[it] * g8[i] + b8[i];
        store8<kBF16>(q.y, static_cast<long long>(row) * q.ldy + col, v);
      }
    }
  }
  cluster_sync_all();      // nobody exits while a peer may still read its statistics
}

template <int BN, bool kBF16, bool kDrop>
static int launch_gemm_ln_t(const GemmParams& p, const LnEpiParams& q, const CUtensorMap& tmA,
                            const CUtensorMap& tmB, cudaStream_t stream) {
  using Cfg = GemmLnCfg<BN>;
  auto kern = gemm_ln_kernel<BN, kBF16, kDrop>;
  static unsigned long long configured = 0;   // per instantiation, one bit per device
  if (first_use_on_device(configured))
    UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  const int grid = p.tiles_m * LN_CLUSTER;
  ProfScope ps(stream);
  UB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), Cfg::SMEM_BYTES, stream, LN_CLUSTER, tmA,
                           tmB, p, q));
  return 0;
}

// N must be 768 (4 x 192) or 1024 (4 x 256); both operands K-major; epilogue = BIAS | RESIDUAL [| DROPOUT].
int launch_gemm_ln(int dtype, const GemmParams& p, const void* gamma, const void* beta, void* y,
                   long long ldy, const CUtensorMap& tmA, const CUtensorMap& tmB, cudaStream_t stream) {
  LnEpiParams q;
  q.gamma = gamma; q.beta = beta; q.y = y; q.ldy = ldy; q.inv_n = 1.0f / static_cast<float>(p.N);
  const bool drop = (p.epilogue & UB200_EPI_DROPOUT) != 0;
  const bool bf = dtype == UB200_BF16;
#define UB_LN_CASE(BNV)                                                                       \
  if (bf) return drop ? launch_gemm_ln_t<BNV, true, true>(p, q, tmA, tmB, stream)             \
                      : launch_gemm_ln_t<BNV, true, false>(p, q, tmA, tmB, stream);           \
  return drop ? launch_gemm_ln_t<BNV, false, true>(p, q, tmA, tmB, stream)                    \
              : launch_gemm_ln_t<BNV, false, false>(p, q, tmA, tmB, stream)
  if (p.N == 768) { UB_LN_CASE(192); }
  if (p.N == 1024) { UB_LN_CASE(256); }
#undef UB_LN_CASE
  return set_error(UB200_EUNSUPPORTED, "gemm+LayerNorm epilogue needs N = 768 or 1024 (got %d)", p.N);
}

}  // namespace ub
