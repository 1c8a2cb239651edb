// wgmma / TMA GEMM core for sm_90a.
//
//   D[M,N] = epilogue( sum_k A[m,k] * B[n,k] ),  16-bit operands, fp32 accumulation in registers.
//
// One persistent CTA per SM, four warpgroups with fixed roles:
//   warpgroup 0     TMA producer — one lane streams 128xBK A tiles and BNxBK B tiles into a
//                   128B-swizzled smem ring (mbarrier full/empty pairs); the warpgroup gives
//                   most of its registers to the consumers (setmaxnreg)
//   warpgroups 1-2  consumers — each owns 64 rows of the 128 x BN tile: 4 x wgmma m64nBNk16 per
//                   stage, a stage is released once the next stage's wgmma group is in flight;
//                   then the finished accumulators go to shared memory, 64 columns at a time, into
//                   a ring of EPI_CHUNKS fp32 chunks (mbarrier full/empty pairs), and the consumers
//                   start the next tile's mainloop
//   warpgroup 3     epilogue — drains each chunk: bias / dropout / residual / GELU / dGELU /
//                   accumulate / column-sum, 16-byte stores
// So the epilogue of one tile runs under the mainloop of the next: a 128-wide tile fits the ring
// whole, wider tiles wait for the first chunks to drain.  The epilogue is the same fp32 code on the
// same fp32 values as a register epilogue would run, so the output bits do not depend on the ring.
//
// kCluster = 2: a cluster of two CTAs on neighbouring 128-row tiles of the same BN columns.  Each
// CTA loads its own A tile and HALF of the B tile, multicast into both CTAs, so every B tile is
// fetched from L2 once per pair.  A slot is refilled only after the consumers of BOTH CTAs have
// released it (they arrive on the empty barrier of both).
//
// Operands may be K-major (contraction dim contiguous; nn.Linear forward) or MN-major
// (contraction dim strided; dgrad reads the weight un-transposed, wgrad reads both activation
// matrices un-transposed) — the wgmma descriptors and transpose bits encode the difference, no transposes are
// ever materialised.  Reference call sites replaced: model/layer.py:76-78,112,140,153 and
// their autograd mirrors.
#pragma once
#include "common.h"
#include "gemm_params.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ub {

constexpr int A_TILE_BYTES = BM * BK * 2;

// Shared-memory layout (gemm_kernel, gemm_group_kernel): the TMA ring, then the ring of fp32
// hand-off chunks (128 rows x 64 columns each), then the mbarriers.  The chunks take the shared
// memory of one TMA stage: 5 stages at BN = 128, 4 at 192, 3 at 256.
constexpr int GEMM_WS_THREADS = 512;    // producer + 2 consumer + epilogue warpgroups
constexpr int CONSUMER_WARPS = 8;       // 16 accumulator rows each; all 8 fill every chunk
constexpr int CHUNK_COLS = 64;
constexpr int CHUNK_BYTES = BM * CHUNK_COLS * 4;
constexpr int EPI_CHUNKS = 2;           // one whole 128-wide tile
constexpr int MAX_DYN_SMEM = 227 * 1024;

template <int BN>
struct WsCfg {
  static constexpr int STAGE_BYTES = A_TILE_BYTES + BN * BK * 2;
  static constexpr int RING_BYTES = EPI_CHUNKS * CHUNK_BYTES;
  static constexpr int BAR_BYTES = 256;
  static constexpr int FIT = (MAX_DYN_SMEM - RING_BYTES - BAR_BYTES - 1024) / STAGE_BYTES;
  static constexpr int STAGES = FIT > 8 ? 8 : FIT;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + RING_BYTES + BAR_BYTES + 1024;  // + align slack
  static_assert((2 * STAGES + 2 * EPI_CHUNKS) * 8 <= BAR_BYTES, "mbarriers overflow their region");
};
static_assert(WsCfg<64>::STAGES == 6 && WsCfg<128>::STAGES == 5 && WsCfg<192>::STAGES == 4 &&
              WsCfg<256>::STAGES == 3, "TMA ring depth per tile width");
static_assert(WsCfg<64>::SMEM_BYTES == 214272 && WsCfg<128>::SMEM_BYTES == 230656 &&
              WsCfg<192>::SMEM_BYTES == 230656 && WsCfg<256>::SMEM_BYTES == 214272,
              "dynamic shared memory per tile width");

template <bool kBF16>
__device__ __forceinline__ void load8(const void* base, long long idx, float (&f)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(
      reinterpret_cast<const typename Elem<kBF16>::T*>(base) + idx));
  float2 t;
  t = Elem<kBF16>::unpack(u.x); f[0] = t.x; f[1] = t.y;
  t = Elem<kBF16>::unpack(u.y); f[2] = t.x; f[3] = t.y;
  t = Elem<kBF16>::unpack(u.z); f[4] = t.x; f[5] = t.y;
  t = Elem<kBF16>::unpack(u.w); f[6] = t.x; f[7] = t.y;
}
template <bool kBF16>
__device__ __forceinline__ void unpack8_(const uint4& u, float (&f)[8]) {
  float2 t;
  t = Elem<kBF16>::unpack(u.x); f[0] = t.x; f[1] = t.y;
  t = Elem<kBF16>::unpack(u.y); f[2] = t.x; f[3] = t.y;
  t = Elem<kBF16>::unpack(u.z); f[4] = t.x; f[5] = t.y;
  t = Elem<kBF16>::unpack(u.w); f[6] = t.x; f[7] = t.y;
}
template <bool kBF16>
__device__ __forceinline__ void store8(void* base, long long idx, const float (&f)[8]) {
  uint4 u;
  u.x = Elem<kBF16>::pack(f[0], f[1]);
  u.y = Elem<kBF16>::pack(f[2], f[3]);
  u.z = Elem<kBF16>::pack(f[4], f[5]);
  u.w = Elem<kBF16>::pack(f[6], f[7]);
  *reinterpret_cast<uint4*>(reinterpret_cast<typename Elem<kBF16>::T*>(base) + idx) = u;
}


// --------------------------------------------------------------------------------- epilogue
// Accumulator register i of the wgmma fragment holds row (lane / 4) + 8 * ((i / 2) % 2) of the
// warp's 16 rows, column 8 * (i / 4) + 2 * (lane % 4) + i % 2.
//
// EPI >= 0 is a compile-time epilogue mask (the combinations the encoder uses are instantiated;
// EPI < 0 falls back to the runtime mask in p.epilogue).
template <int EPI, bool kBF16>
struct EpiMask {
  const int rt;
  __device__ __forceinline__ explicit EpiMask(int runtime) : rt(runtime) {}
  // EPI == -2: runtime mask of the deterministic mode, built without the atomic epilogues
  __device__ __forceinline__ bool has(int bit) const {
    if (EPI == -2 && (bit & (UB200_EPI_COLSUM | UB200_EPI_ATOMIC))) return false;
    return EPI >= 0 ? (EPI & bit) != 0 : (rt & bit) != 0;
  }
};

// Word of element (r, c) in a 128 x 64 fp32 hand-off chunk.  Rows are 64 words; the 16-byte column
// groups are XOR-swizzled by (r & 3) << 1 | (r & 1), so that the consumers' fragment writes (a
// half-warp stores 8-byte pieces of 4 rows) and the epilogue's reads (a quarter-warp loads 16-byte
// pieces of 2 rows) are both free of bank conflicts.
__device__ __forceinline__ int chunk_word(int r, int c) {
  return r * CHUNK_COLS + ((((c >> 2) ^ (((r & 3) << 1) | (r & 1)))) << 2) + (c & 3);
}

// Consumer warp: columns [64 c, 64 c + 64) of its 16 accumulator rows [r0, r0 + 16) into `chunk`.
template <int BN>
__device__ __forceinline__ void stage_chunk(const float (&acc)[BN / 2], int c, int r0, int lane, float* chunk) {
#pragma unroll
  for (int t = 0; t < 32; t += 2) {
    const int r = r0 + (lane >> 2) + 8 * ((t >> 1) & 1);
    const int cc = 8 * (t >> 2) + 2 * (lane & 3);
    *reinterpret_cast<float2*>(chunk + chunk_word(r, cc)) = make_float2(acc[32 * c + t], acc[32 * c + t + 1]);
  }
}

// Consumer warp `cw` (0..7): hand the finished tile to the epilogue warpgroup, one chunk per 64
// columns (columns at or beyond N are never written, and no chunk is sent for them).
template <int BN>
__device__ __forceinline__ void handoff_tile(const float (&acc)[BN / 2], int n0, int N, int cw, int lane, float* ring,
                                             uint64_t* chunk_full, uint64_t* chunk_empty, int& cs, uint32_t& cphase) {
#pragma unroll
  for (int c = 0; c < BN / CHUNK_COLS; ++c) {
    if (n0 + c * CHUNK_COLS >= N) break;
    mbar_wait(&chunk_empty[cs], cphase ^ 1);
    stage_chunk<BN>(acc, c, 16 * cw, lane, ring + cs * (CHUNK_BYTES / 4));
    __syncwarp();
    if (lane == 0) mbar_arrive(&chunk_full[cs]);
    if (++cs == EPI_CHUNKS) { cs = 0; cphase ^= 1; }
  }
}

// Epilogue warp `ew` (0..3): rows [m0 + 32 ew, m0 + 32 ew + 32) x columns [c0, c0 + 64) of the tile,
// read from `chunk` once `full` completes its phase `parity`.  4 lanes own one row in 8-column
// pieces: every global access of the warp covers 8 rows x 64 contiguous bytes and the column sum
// needs 3 shuffle steps.  The side inputs (bias / residual / dGELU aux / accumulate) of the chunk
// are requested before it is waited for.
template <int EPI, bool kBF16>
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, int m0, int c0, int ew, int lane,
                                               const DropoutRng& rng, const float* chunk, uint64_t* full,
                                               uint32_t parity) {
  using T16 = typename Elem<kBF16>::T;
  const EpiMask<EPI, kBF16> E(p.epilogue);
  const int sub_r = lane >> 2;        // row inside an 8-row group
  const int cg = (lane & 3) * 8;      // first of this lane's 8 columns inside a 32-column block
  const bool side16 = E.has(UB200_EPI_RESIDUAL) || E.has(UB200_EPI_DGELU) ||
                      (E.has(UB200_EPI_ACCUM) && !E.has(UB200_EPI_OUT_F32));
  const T16* side_base = E.has(UB200_EPI_RESIDUAL) ? reinterpret_cast<const T16*>(p.residual)
                         : (E.has(UB200_EPI_DGELU) ? reinterpret_cast<const T16*>(p.aux)
                                                   : reinterpret_cast<const T16*>(p.out));
  const long long side_ld = E.has(UB200_EPI_RESIDUAL) ? p.ldr : (E.has(UB200_EPI_DGELU) ? p.ldaux : p.ldo);
  uint4 bias4[2], side[2][4];
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int col = c0 + 32 * b + cg;
    bias4[b] = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int it = 0; it < 4; ++it) side[b][it] = make_uint4(0, 0, 0, 0);
    if (col < p.N) {                  // N % 8 == 0 is enforced on the host
      if (E.has(UB200_EPI_BIAS))
        bias4[b] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.bias) + col));
      if (side16) {
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int row = m0 + 32 * ew + it * 8 + sub_r;
          if (row < p.M)
            side[b][it] = __ldg(reinterpret_cast<const uint4*>(side_base + static_cast<long long>(row) * side_ld + col));
        }
      }
    }
  }
  mbar_wait(full, parity);

#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const int col0 = c0 + 32 * b;
    if (col0 >= p.N) break;           // warp-uniform
    const int col = col0 + cg;
    const bool col_ok = col < p.N;
    float bias8[8];
    unpack8_<kBF16>(bias4[b], bias8);
    float csum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) csum[i] = 0.f;

#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int rr = 32 * ew + it * 8 + sub_r;
      const int row = m0 + rr;
      const float4 lo = *reinterpret_cast<const float4*>(chunk + chunk_word(rr, 32 * b + cg));
      const float4 hi = *reinterpret_cast<const float4*>(chunk + chunk_word(rr, 32 * b + cg + 4));
      const float a8[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = a8[i] + bias8[i];
      if (!(col_ok && row < p.M)) continue;
      if (E.has(UB200_EPI_DROPOUT)) {
        const uint64_t e = static_cast<uint64_t>(row) * static_cast<uint64_t>(p.N) + col;
        const uint4 rnd = rng.draw8(e >> 3);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = (rand16_of(rnd, i) < rng.thr16) ? 0.f : v[i] * rng.inv_keep;
      }
      if (E.has(UB200_EPI_RESIDUAL)) {
        float t[8];
        unpack8_<kBF16>(side[b][it], t);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] += t[i];
      }
      if (E.has(UB200_EPI_GELU)) {
        float pre[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          // the reference rounds the Linear output to 16 bits before GELU
          pre[i] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(v[i]));
          v[i] = gelu_erf(pre[i]);
        }
        store8<kBF16>(p.out2, static_cast<long long>(row) * p.ldo + col, pre);
      }
      if (E.has(UB200_EPI_TANH)) {       // generic (runtime-mask) kernel only
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = tanhf(v[i]);
      }
      if (E.has(UB200_EPI_DGELU)) {
        float t[8];
        if (E.has(UB200_EPI_RESIDUAL))   // generic path only: aux was not prefetched
          load8<kBF16>(p.aux, static_cast<long long>(row) * p.ldaux + col, t);
        else
          unpack8_<kBF16>(side[b][it], t);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] *= dgelu_erf(t[i]);
      }
      if (E.has(UB200_EPI_OUT_F32)) {
        float* o = reinterpret_cast<float*>(p.out) + static_cast<long long>(row) * p.ldo + col;
        if (E.has(UB200_EPI_ACCUM)) {
          const float4 o0 = *reinterpret_cast<const float4*>(o);
          const float4 o1 = *reinterpret_cast<const float4*>(o + 4);
          v[0] += o0.x; v[1] += o0.y; v[2] += o0.z; v[3] += o0.w;
          v[4] += o1.x; v[5] += o1.y; v[6] += o1.z; v[7] += o1.w;
        }
        if (E.has(UB200_EPI_ATOMIC)) {     // split-K partial sums meet in a pre-zeroed fp32 output
#pragma unroll
          for (int i = 0; i < 8; ++i) atomicAdd(o + i, v[i]);
        } else {
          *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
          *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
        }
      } else {
        if (E.has(UB200_EPI_ACCUM)) {
          float t[8];
          if (E.has(UB200_EPI_RESIDUAL) || E.has(UB200_EPI_DGELU))
            load8<kBF16>(p.out, static_cast<long long>(row) * p.ldo + col, t);   // generic path
          else
            unpack8_<kBF16>(side[b][it], t);
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] += t[i];
        }
        store8<kBF16>(p.out, static_cast<long long>(row) * p.ldo + col, v);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) csum[i] += v[i];
    }
    if (E.has(UB200_EPI_COLSUM)) {
      // lanes with equal (lane & 3) own the same 8 columns: reduce over the 8 row-lanes
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float x = csum[i];
        x += __shfl_xor_sync(0xffffffffu, x, 4);
        x += __shfl_xor_sync(0xffffffffu, x, 8);
        x += __shfl_xor_sync(0xffffffffu, x, 16);
        csum[i] = x;
      }
      if (lane < 4 && col_ok) {        // two 16-byte vector atomics instead of eight scalar ones
        atomicAdd(reinterpret_cast<float4*>(p.colsum + col), make_float4(csum[0], csum[1], csum[2], csum[3]));
        atomicAdd(reinterpret_cast<float4*>(p.colsum + col + 4), make_float4(csum[4], csum[5], csum[6], csum[7]));
      }
    }
  }
}


__device__ __forceinline__ DropoutRng make_rng(const GemmParams& p) {
  DropoutRng rng;
  rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = p.stream_lo; rng.s1 = p.stream_hi;
  if (p.epilogue & UB200_EPI_DROPOUT) rng_add_dev_offset(p.rng_dev, rng.s0, rng.s1);
  rng.thr16 = p.drop_thr16; rng.inv_keep = p.drop_inv_keep;
  return rng;
}

// 512-thread kernels start at 128 registers a thread: 24 + 2 x 192 + 104 = 4 x 128
__device__ __forceinline__ void setmaxnreg_ws_producer() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
}
__device__ __forceinline__ void setmaxnreg_ws_consumer() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 192;" ::: "memory");
}
__device__ __forceinline__ void setmaxnreg_ws_epilogue() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 104;" ::: "memory");
}

// ------------------------------------------------------------------------------ pipeline halves
// Producer lane: k-blocks [kb0, kb1) of the 128 x BN tile at (m0, n0) into the ring.  With
// kCluster = 2 this CTA (cluster rank `rank`) loads half of the B tile and multicasts it.
template <int BN, bool A_MN, bool B_MN, int kCluster>
__device__ __forceinline__ void produce_tile(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                             const CUtensorMap* tmA, const CUtensorMap* tmB, int m0, int n0,
                                             int kb0, int kb1, int& stage, uint32_t& phase, uint32_t rank) {
  using Cfg = WsCfg<BN>;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&empty_bar[stage], phase ^ 1);
    uint8_t* sA = smem + stage * Cfg::STAGE_BYTES;
    uint8_t* sB = sA + A_TILE_BYTES;
    mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);   // own A + the whole B tile
    if (!A_MN) {
      tma_load_2d(sA, tmA, &full_bar[stage], kb * BK, m0);
    } else {
#pragma unroll
      for (int j = 0; j < BM / 64; ++j)
        tma_load_2d(sA + j * (64 * BK * 2), tmA, &full_bar[stage], m0 + j * 64, kb * BK);
    }
    if (kCluster == 1) {
      if (!B_MN) {
        tma_load_2d(sB, tmB, &full_bar[stage], kb * BK, n0);
      } else {
#pragma unroll
        for (int j = 0; j < BN / 64; ++j)
          tma_load_2d(sB + j * (64 * BK * 2), tmB, &full_bar[stage], n0 + j * 64, kb * BK);
      }
    } else {
      constexpr int BH = BN / 2;
      if (!B_MN) {
        tma_load_2d_mc(sB + rank * (BH * BK * 2), tmB, &full_bar[stage], kb * BK, n0 + rank * BH, 3);
      } else {
#pragma unroll
        for (int j = 0; j < BH / 64; ++j) {
          const int jj = rank * (BH / 64) + j;
          tma_load_2d_mc(sB + jj * (64 * BK * 2), tmB, &full_bar[stage], n0 + jj * 64, kb * BK, 3);
        }
      }
    }
    if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
  }
}

// Consumer warpgroup `wg` (rows [64 wg, 64 wg + 64) of the tile): acc = A B^T over nkb k-blocks.
// K-major operands advance 16 elements = 32 B inside the swizzle row per k16 step; MN-major ones
// advance 16 K-rows = 2048 B, their 64-wide M/N groups are one 8 KB box apart.
template <int BN, bool A_MN, bool B_MN, bool kBF16, int kCluster>
__device__ __forceinline__ void consume_tile(float (&acc)[BN / 2], uint8_t* smem, uint64_t* full_bar,
                                             uint64_t* empty_bar, int nkb, int wg, int& stage,
                                             uint32_t& phase, uint32_t peer) {
  using Cfg = WsCfg<BN>;
  constexpr uint32_t A_KSTEP = A_MN ? 2048 : 32, A_LBO = A_MN ? 8192 : 16;
  constexpr uint32_t B_KSTEP = B_MN ? 2048 : 32, B_LBO = B_MN ? 8192 : 16;
  const bool releaser = (threadIdx.x & 127) == 0;
  int prev = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sA = smem_u32(smem + stage * Cfg::STAGE_BYTES) + wg * (64 * 128);
    const uint32_t sB = smem_u32(smem + stage * Cfg::STAGE_BYTES) + A_TILE_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
      const uint64_t da = gmma_desc(sA + k * A_KSTEP, A_LBO, 1024);
      const uint32_t scale_d = (kb | k) != 0 ? 1u : 0u;
      if constexpr (BN == 256) {
        // two m64n128 halves (columns 128.. start 16 KB into the B tile, K- or MN-major): an m64n256
        // wgmma needs more than the 128 registers a thread of a 512-thread kernel launches with.
        // The fragment layout, and every output bit, is that of the m64n256 form.
        float (&lo)[64] = *reinterpret_cast<float(*)[64]>(&acc[0]);
        float (&hi)[64] = *reinterpret_cast<float(*)[64]>(&acc[64]);
        Wgmma<128, kBF16, A_MN, B_MN>::ss(lo, da, gmma_desc(sB + k * B_KSTEP, B_LBO, 1024), scale_d);
        Wgmma<128, kBF16, A_MN, B_MN>::ss(hi, da, gmma_desc(sB + 128 * 128 + k * B_KSTEP, B_LBO, 1024), scale_d);
      } else {
        Wgmma<BN, kBF16, A_MN, B_MN>::ss(acc, da, gmma_desc(sB + k * B_KSTEP, B_LBO, 1024), scale_d);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();                   // the previous stage's wgmma group has retired
    if (prev >= 0 && releaser) {
      mbar_arrive(&empty_bar[prev]);
      if (kCluster == 2) mbar_arrive_cluster(mapa_shared(smem_u32(&empty_bar[prev]), peer));
    }
    prev = stage;
    if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (releaser) {
    mbar_arrive(&empty_bar[prev]);
    if (kCluster == 2) mbar_arrive_cluster(mapa_shared(smem_u32(&empty_bar[prev]), peer));
  }
}

// ============================================================ epilogue-warpgroup kernels: layout
// WsCfg's carve-up of the (1024-aligned) dynamic shared memory.  Thread 0 initialises the barriers:
// a TMA stage is emptied by the consumer warpgroups (of both CTAs with kCluster = 2), a chunk is
// filled by the 8 consumer warps and emptied by the 4 epilogue warps.
template <int BN>
struct WsSmem {
  using Cfg = WsCfg<BN>;
  float* ring;
  uint64_t* full_bar;
  uint64_t* empty_bar;
  uint64_t* chunk_full;
  uint64_t* chunk_empty;
  __device__ __forceinline__ explicit WsSmem(uint8_t* smem)
      : ring(reinterpret_cast<float*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES)),
        full_bar(reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES + Cfg::RING_BYTES)),
        empty_bar(full_bar + Cfg::STAGES),
        chunk_full(empty_bar + Cfg::STAGES),
        chunk_empty(chunk_full + EPI_CHUNKS) {}
  __device__ __forceinline__ void init(int kCluster) const {
    for (int s = 0; s < Cfg::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * kCluster);
    }
    for (int s = 0; s < EPI_CHUNKS; ++s) {
      mbar_init(&chunk_full[s], CONSUMER_WARPS);
      mbar_init(&chunk_empty[s], 4);
    }
    fence_barrier_init();
  }
  // epilogue warp `ew`: the chunks of the tile at (m0, n0), in the order handoff_tile sends them
  template <int EPI, bool kBF16>
  __device__ __forceinline__ void drain_tile(const GemmParams& p, int m0, int n0, int ew, int lane,
                                             const DropoutRng& rng, int& cs, uint32_t& cphase) const {
    for (int c0 = n0; c0 < n0 + BN && c0 < p.N; c0 += CHUNK_COLS) {
      epilogue_chunk<EPI, kBF16>(p, m0, c0, ew, lane, rng, ring + cs * (CHUNK_BYTES / 4), &chunk_full[cs], cphase);
      __syncwarp();
      if (lane == 0) mbar_arrive(&chunk_empty[cs]);
      if (++cs == EPI_CHUNKS) { cs = 0; cphase ^= 1; }
    }
  }
};

// =================================================================================== GEMM kernel
template <int BN, bool A_MN, bool B_MN, bool kBF16, int kCluster, int EPI>
__global__ void __launch_bounds__(GEMM_WS_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
            const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment.  The offset is computed in the shared window
  // and applied by pointer arithmetic on the __shared__ array so that the compiler keeps the
  // shared address space (STS / LDS instead of generic ST / LD).
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const WsSmem<BN> sm(smem);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = kCluster == 2 ? cluster_ctarank() : 0u;
  const int num_kb = (p.K + BK - 1) / BK;
  const int num_tiles = p.tiles_n * (kCluster == 2 ? (p.tiles_m + 1) / 2 : p.tiles_m);
  // work unit = (tile, k-slice): unit % num_tiles is the tile, unit / num_tiles the slice of
  // kb_per_split k-blocks (ksplit == 1: one slice covering all of K).  A cluster pair shares one
  // unit sequence; its tile is 256 rows high.
  const int num_units = num_tiles * p.ksplit;
  const int unit0 = kCluster == 2 ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  const int unit_step = kCluster == 2 ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    sm.init(kCluster);
  }
  pdl_launch_dependents();   // dependents may start their own prologue
  __syncthreads();
  if (kCluster == 2) cluster_sync_all();   // both CTAs' barriers exist before any multicast / remote arrive
  pdl_wait();                // the producing kernel has completed; its outputs are visible

  if (warp < 4) {
    setmaxnreg_ws_producer();
    // ===================================================================== TMA producer
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = unit0; unit < num_units; unit += unit_step) {
        const int tile = unit % num_tiles;
        const int kb0 = (unit / num_tiles) * p.kb_per_split;
        const int kb1 = min(num_kb, kb0 + p.kb_per_split);
        const int m0 = (tile / p.tiles_n) * (kCluster * BM) + static_cast<int>(rank) * BM;
        const int n0 = (tile % p.tiles_n) * BN;
        produce_tile<BN, A_MN, B_MN, kCluster>(smem, sm.full_bar, sm.empty_bar, &tmA, &tmB, m0, n0,
                                               kb0, kb1, stage, phase, rank);
      }
    }
  } else if (warp < 12) {
    setmaxnreg_ws_consumer();
    // ===================================================================== consumers
    const int cw = warp - 4;              // consumer warp 0..7: tile rows [16 cw, 16 cw + 16)
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, cs = 0;
    uint32_t phase = 0, cphase = 0;
    for (int unit = unit0; unit < num_units; unit += unit_step) {
      const int tile = unit % num_tiles;
      const int kb0 = (unit / num_tiles) * p.kb_per_split;
      const int kb1 = min(num_kb, kb0 + p.kb_per_split);
      const int n0 = (tile % p.tiles_n) * BN;
      consume_tile<BN, A_MN, B_MN, kBF16, kCluster>(acc, smem, sm.full_bar, sm.empty_bar,
                                                    kb1 - kb0, cw >> 2, stage, phase, rank ^ 1u);
      handoff_tile<BN>(acc, n0, p.N, cw, lane, sm.ring, sm.chunk_full, sm.chunk_empty, cs, cphase);
    }
  } else {
    setmaxnreg_ws_epilogue();
    // ===================================================================== epilogue
    const int ew = warp - 12;             // epilogue warp 0..3: tile rows [32 ew, 32 ew + 32)
    const DropoutRng rng = make_rng(p);
    int cs = 0;
    uint32_t cphase = 0;
    for (int unit = unit0; unit < num_units; unit += unit_step) {
      const int tile = unit % num_tiles;
      const int m0 = (tile / p.tiles_n) * (kCluster * BM) + static_cast<int>(rank) * BM;
      const int n0 = (tile % p.tiles_n) * BN;
      sm.template drain_tile<EPI, kBF16>(p, m0, n0, ew, lane, rng, cs, cphase);
    }
  }
  if (kCluster == 2) cluster_sync_all();   // nobody exits while the peer may still signal it
}

// =================================================================================== grouped wgrad
// The four weight-gradient GEMMs of a layer (dW2 = dY2^T f, dW1 = dPre^T a, dWo = dY1^T ctx,
// dWqkv = dQKV^T x; all contract over K = T tokens, both operands MN-major) as ONE persistent
// launch instead of four, each with its own prologue and exposed epilogue tail.
struct TmPack {
  CUtensorMap a[GEMM_MAX_GROUP];
  CUtensorMap b[GEMM_MAX_GROUP];
};

__device__ __forceinline__ int group_of_tile(const GroupedParams& g, int tile) {
  int pi = 0;
#pragma unroll
  for (int i = 1; i < GEMM_MAX_GROUP; ++i)
    if (i < g.nprob && tile >= g.tile_start[i]) pi = i;
  return pi;
}

template <int BN, bool kBF16, int EPI>
__global__ void __launch_bounds__(GEMM_WS_THREADS, 1)
gemm_group_kernel(const __grid_constant__ TmPack tm, const GroupedParams g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const WsSmem<BN> sm(smem);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = (g.K + BK - 1) / BK;
  const int num_tiles = g.tile_start[g.nprob];

  if (warp == 0 && lane == 0) sm.init(1);
  pdl_launch_dependents();
  __syncthreads();
  pdl_wait();

  if (warp < 4) {
    setmaxnreg_ws_producer();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int pi = group_of_tile(g, tile);
        const int lt = tile - g.tile_start[pi];
        const int m0 = (lt / g.tiles_n[pi]) * BM;
        const int n0 = (lt % g.tiles_n[pi]) * BN;
        produce_tile<BN, true, true, 1>(smem, sm.full_bar, sm.empty_bar, &tm.a[pi], &tm.b[pi], m0, n0,
                                        0, num_kb, stage, phase, 0u);
      }
    }
  } else if (warp < 12) {
    setmaxnreg_ws_consumer();
    const int cw = warp - 4;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, cs = 0;
    uint32_t phase = 0, cphase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int pi = group_of_tile(g, tile);
      const int lt = tile - g.tile_start[pi];
      const int n0 = (lt % g.tiles_n[pi]) * BN;
      consume_tile<BN, true, true, kBF16, 1>(acc, smem, sm.full_bar, sm.empty_bar, num_kb,
                                             cw >> 2, stage, phase, 0u);
      handoff_tile<BN>(acc, n0, g.N[pi], cw, lane, sm.ring, sm.chunk_full, sm.chunk_empty, cs, cphase);
    }
  } else {
    setmaxnreg_ws_epilogue();
    const int ew = warp - 12;
    DropoutRng rng;
    rng.k0 = rng.k1 = rng.s0 = rng.s1 = 0; rng.thr16 = 0; rng.inv_keep = 1.f;
    int cs = 0;
    uint32_t cphase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int pi = group_of_tile(g, tile);
      const int lt = tile - g.tile_start[pi];
      const int m0 = (lt / g.tiles_n[pi]) * BM;
      const int n0 = (lt % g.tiles_n[pi]) * BN;
      GemmParams pp{};
      pp.M = g.M[pi]; pp.N = g.N[pi]; pp.K = g.K; pp.epilogue = g.epilogue;
      pp.out = g.out[pi]; pp.ldo = g.ldo[pi];
      sm.template drain_tile<EPI, kBF16>(pp, m0, n0, ew, lane, rng, cs, cphase);
    }
  }
}

template <int BN, bool A_MN, bool B_MN, bool kBF16, int kCluster, int EPI>
static int launch_gemm(const GemmParams& p, const CUtensorMap& tmA, const CUtensorMap& tmB, int grid,
                       cudaStream_t stream) {
  using Cfg = WsCfg<BN>;
  void (*kern)(const CUtensorMap, const CUtensorMap, const GemmParams) = gemm_kernel<BN, A_MN, B_MN, kBF16, kCluster, EPI>;
  static unsigned long long configured = 0;  // per instantiation, one bit per device
  if (first_use_on_device(configured))
    UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Cfg::SMEM_BYTES));
  {
    ProfScope ps(stream);
    UB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(GEMM_WS_THREADS), Cfg::SMEM_BYTES, stream, kCluster,
                             tmA, tmB, p));
  }
  return 0;
}

// Epilogue masks the encoder uses get their own instantiation (per operand-major form); any
// other mask runs the runtime-flag kernel (EPI = -1, or -2 in deterministic mode).
template <int BN, bool kBF16, int kCluster>
static int dispatch_major(int a_major, int b_major, const GemmParams& p, const CUtensorMap& tmA,
                          const CUtensorMap& tmB, int grid, cudaStream_t stream) {
  const int e = p.epilogue;
  const bool det = deterministic();
#define UB_CASE(AMN, BMN, MASK) \
  if (e == (MASK)) return launch_gemm<BN, AMN, BMN, kBF16, kCluster, (MASK)>(p, tmA, tmB, grid, stream)
#define UB_GENERIC(AMN, BMN)                                                                      \
  return det ? launch_gemm<BN, AMN, BMN, kBF16, kCluster, -2>(p, tmA, tmB, grid, stream)         \
             : launch_gemm<BN, AMN, BMN, kBF16, kCluster, -1>(p, tmA, tmB, grid, stream)
  if (a_major == 0 && b_major == 0) {            // forward nn.Linear
    UB_CASE(false, false, UB200_EPI_BIAS);
    UB_CASE(false, false, UB200_EPI_BIAS | UB200_EPI_GELU);
    UB_CASE(false, false, UB200_EPI_BIAS | UB200_EPI_RESIDUAL);
    UB_CASE(false, false, UB200_EPI_BIAS | UB200_EPI_DROPOUT | UB200_EPI_RESIDUAL);
    UB_GENERIC(false, false);
  }
  if (a_major == 0 && b_major == 1) {            // dgrad
    UB_CASE(false, true, 0);
    UB_CASE(false, true, UB200_EPI_RESIDUAL);
    UB_CASE(false, true, UB200_EPI_DGELU | UB200_EPI_COLSUM);
    if (det) UB_CASE(false, true, UB200_EPI_DGELU);   // DGELU | COLSUM of the deterministic mode
    UB_GENERIC(false, true);
  }
  if (a_major == 1 && b_major == 1) {            // wgrad
    UB_CASE(true, true, 0);
    UB_CASE(true, true, UB200_EPI_ACCUM);
    UB_GENERIC(true, true);
  }
#undef UB_GENERIC
#undef UB_CASE
  return set_error(UB200_EUNSUPPORTED, "gemm: a_major=1 with b_major=0 is not instantiated");
}

template <bool kBF16>
int gemm_dispatch(int bn, int cluster, int a_major, int b_major, const GemmParams& p,
                  const CUtensorMap& tmA, const CUtensorMap& tmB, int grid, cudaStream_t stream) {
  if (cluster == 2) {
    switch (bn) {
      case 128: return dispatch_major<128, kBF16, 2>(a_major, b_major, p, tmA, tmB, grid, stream);
      case 256: return dispatch_major<256, kBF16, 2>(a_major, b_major, p, tmA, tmB, grid, stream);
    }
    return set_error(UB200_EINVAL, "gemm: cluster 2 needs tile_n 128 or 256 (got %d)", bn);
  }
  switch (bn) {
    case 64: return dispatch_major<64, kBF16, 1>(a_major, b_major, p, tmA, tmB, grid, stream);
    case 128: return dispatch_major<128, kBF16, 1>(a_major, b_major, p, tmA, tmB, grid, stream);
    case 192: return dispatch_major<192, kBF16, 1>(a_major, b_major, p, tmA, tmB, grid, stream);
    case 256: return dispatch_major<256, kBF16, 1>(a_major, b_major, p, tmA, tmB, grid, stream);
  }
  return set_error(UB200_EINVAL, "gemm: tile_n must be 0, 64, 128, 192 or 256 (got %d)", bn);
}

template <int BN, bool kBF16>
int gemm_group_launch(const TmPack& tm, const GroupedParams& g, int grid, cudaStream_t stream) {
  using Cfg = WsCfg<BN>;
  void (*kern)(const TmPack, const GroupedParams);
  if (g.epilogue == 0) kern = gemm_group_kernel<BN, kBF16, 0>;
  else if (g.epilogue == UB200_EPI_ACCUM) kern = gemm_group_kernel<BN, kBF16, UB200_EPI_ACCUM>;
  else return set_error(UB200_EUNSUPPORTED, "gemm_grouped: epilogue must be 0 or ACCUM");
  static unsigned long long configured[2] = {0, 0};   // per instantiation, one bit per device
  const int ci = g.epilogue ? 1 : 0;
  if (first_use_on_device(configured[ci]))
    UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  ProfScope ps(stream);
  UB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(GEMM_WS_THREADS), Cfg::SMEM_BYTES, stream, 1, tm, g));
  return 0;
}

template <bool kBF16>
int gemm_group_dispatch(const TmPack& tm, const GroupedParams& g, int grid, cudaStream_t stream) {
  switch (g.bn) {
    case 128: return gemm_group_launch<128, kBF16>(tm, g, grid, stream);
    case 192: return gemm_group_launch<192, kBF16>(tm, g, grid, stream);
    case 256: return gemm_group_launch<256, kBF16>(tm, g, grid, stream);
  }
  return set_error(UB200_EINVAL, "gemm_grouped: tile_n must be 128, 192 or 256 (got %d)", g.bn);
}

}  // namespace ub
