// HBM-bound row-wise kernels of the encoder path (16-byte vector loads, fp32 statistics):
//   ln_fwd        y = LayerNorm(x) * gamma + beta              (apex FusedLayerNorm semantics:
//                 biased variance, eps inside the sqrt — model/layer.py:108,114,149,155)
//   ln_bwd        dx (and dropout-masked dx), dgamma, dbeta, column-sum of the masked dx
//                 (= bias gradient of the Linear that fed the residual sum), one pass
//   ReLU rows     y = LayerNorm(relu(pre)) and its backward (dpre = dx o (pre > 0) in the masked-output
//                 slot): the Linear(H, 2H) -> ReLU -> LayerNorm(2H) prefix of the VCR head (model/vcr.py)
//   gather_rows   dst[r] = idx[r] >= 0 ? src[idx[r]] : 0     (pack / unpack between the padded
//                 [B, L, H] view of the reference API and the packed [T, H] layout; bit-exact)
//   colsum        out[n] += sum_m x[m, n]                       (bias gradient of the QKV projection)
//   cvt           16-bit <- fp32 (+ optional accumulate): small-gradient finalisation
// One warp per row; a lane owns the same columns in every row it visits so that the column
// reductions of ln_bwd stay in registers until one smem + atomic step per CTA.
#include "common.h"
#include "ptx.cuh"

namespace ub {

constexpr int LN_MAX_VEC = 4;  // per lane: 4 x 8 columns -> H <= 1024
// Rows wider than 1024 columns (up to 2048) and ReLU-input rows run their own instantiations with
// NV = 4, 6 or 8 vectors per lane (ln_wide_nv); the H <= 1024 plain-row kernels are left as they are.
constexpr int LN_WIDE_MAX_VEC = 8;  // H <= 2048
__host__ __device__ constexpr int ln_wide_nv(int H) {
  return H <= 4 * 256 ? 4 : (H <= 6 * 256 ? 6 : 8);
}
constexpr float LN_EPS = 1e-12f;

template <bool kBF16>
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  float2 t;
  t = Elem<kBF16>::unpack(u.x); f[0] = t.x; f[1] = t.y;
  t = Elem<kBF16>::unpack(u.y); f[2] = t.x; f[3] = t.y;
  t = Elem<kBF16>::unpack(u.z); f[4] = t.x; f[5] = t.y;
  t = Elem<kBF16>::unpack(u.w); f[6] = t.x; f[7] = t.y;
}
template <bool kBF16>
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  u.x = Elem<kBF16>::pack(f[0], f[1]); u.y = Elem<kBF16>::pack(f[2], f[3]);
  u.z = Elem<kBF16>::pack(f[4], f[5]); u.w = Elem<kBF16>::pack(f[6], f[7]);
  return u;
}
// relu of eight packed 16-bit values (fp16 or bf16: the sign is bit 15): every value with the sign bit
// set becomes +0, the others are kept bit for bit.
__device__ __forceinline__ uint32_t relu16x2(uint32_t u) {
  return u & ~(((u >> 15) & 0x00010001u) * 0xFFFFu);
}
__device__ __forceinline__ uint4 relu16x8(uint4 u) {
  return make_uint4(relu16x2(u.x), relu16x2(u.y), relu16x2(u.z), relu16x2(u.w));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------ LayerNorm fwd
// kRelu: y = LayerNorm(relu(x)); relu of a 16-bit value is exact, so the statistics see exactly the
// values torch's ReLU would hand to the LayerNorm.  (The ReLU instantiations state a minimum of one CTA
// per SM: with no minimum, ptxas keeps them at 48-80 registers and spills.)
template <bool kBF16, int NV = LN_MAX_VEC, bool kRelu = false>
__global__ void __launch_bounds__(256, kRelu ? 1 : 0)
ln_fwd_kernel(const void* __restrict__ x_, const void* __restrict__ gamma_,
              const void* __restrict__ beta_, void* __restrict__ y_, int rows, int H) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + warp;
  if (row >= rows) return;
  const int nvec = H >> 3;
  const uint4* x = reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(x_) +
                                                  static_cast<size_t>(row) * H);
  float v[NV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      unpack8<kBF16>(kRelu ? relu16x8(__ldg(x + vi)) : __ldg(x + vi), v[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) sum += v[i][e];
    }
  }
  const float mean = warp_sum(sum) / H;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = v[i][e] - mean; sq += d * d; }
    }
  const float rstd = rsqrtf(warp_sum(sq) / H + LN_EPS);
  const uint4* g = reinterpret_cast<const uint4*>(gamma_);
  const uint4* bt = reinterpret_cast<const uint4*>(beta_);
  uint4* y = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(y_) + static_cast<size_t>(row) * H);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float gg[8], bb[8], o[8];
      unpack8<kBF16>(__ldg(g + vi), gg);
      unpack8<kBF16>(__ldg(bt + vi), bb);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * gg[e] + bb[e];
      y[vi] = pack8<kBF16>(o);
    }
  }
}

// ------------------------------------------------------------------------------ LayerNorm bwd
struct LnBwdParams {
  const void* dy;      // [rows, H]
  const void* x;       // [rows, H]  pre-LN sum saved by the forward
  const void* gamma;   // [H]
  void* dx;            // [rows, H]  gradient wrt the pre-LN sum (residual branch)
  void* dx_drop;       // [rows, H]  dx o dropout-mask / keep (Linear branch); NULL if p == 0
  float* dgamma;       // [H] fp32, atomically accumulated
  float* dbeta;        // [H]
  float* dbias;        // [H] column sum of the Linear-branch gradient; may be NULL
  int rows, H;
  uint32_t drop_thr16;
  float drop_inv_keep;
  uint32_t seed_lo, seed_hi, stream_lo, stream_hi;
  const int* row_kind;  // optional [rows]: only rows with row_kind[row] == kind take part
  int kind;
  int dy_drop;          // 1: the dropout mask applies to dy (y = dropout(LN(x)), embeddings)
  int zero_inactive;    // 1: rows of the other kind get dx = 0 (instead of being left untouched)
  const unsigned long long* rng_dev;   // optional device-side dropout stream offset (graph replay)
};

// NV = vectors (8 columns) per lane = ceil(H / 256): register arrays are sized for the actual
// hidden size (H = 768 -> 3), and the next row's x / dy are prefetched while the current row is
// reduced, so one wave of one CTA per SM covers the whole [T, H] matrix.
template <bool kBF16, int NV>
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const LnBwdParams p) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  __shared__ float red[3][8][32 * 8 + 1];  // [quantity][warp][lane*8+e] for one vector slot
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nwarps = blockDim.x >> 5;
  const int H = p.H, nvec = H >> 3;
  float gam[NV][8];
  float acc_g[NV][8], acc_b[NV][8], acc_d[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
#pragma unroll
    for (int e = 0; e < 8; ++e) { gam[i][e] = 0.f; acc_g[i][e] = 0.f; acc_b[i][e] = 0.f; acc_d[i][e] = 0.f; }
    if (vi < nvec) unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.gamma) + vi), gam[i]);
  }
  DropoutRng rng;
  rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = p.stream_lo; rng.s1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rng.s0, rng.s1);
  rng.thr16 = p.drop_thr16; rng.inv_keep = p.drop_inv_keep;
  const float inv_h = 1.0f / H;

  const int stride = gridDim.x * nwarps;
  int row = blockIdx.x * nwarps + warp;
  uint4 nx[NV], nd[NV];
  if (row < p.rows) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        nx[i] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.x) +
                                                     static_cast<size_t>(row) * H) + vi);
        nd[i] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.dy) +
                                                     static_cast<size_t>(row) * H) + vi);
      }
    }
  }
  for (; row < p.rows; row += stride) {
    float xv[NV][8], dv[NV][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (lane + i * 32 < nvec) {
        unpack8<kBF16>(nx[i], xv[i]);
        unpack8<kBF16>(nd[i], dv[i]);
#pragma unroll
        for (int e = 0; e < 8; ++e) sum += xv[i][e];
      }
    }
    if (p.dy_drop) {                 // y = dropout(LN(x)): mask the incoming gradient
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int vi = lane + i * 32;
        if (vi < nvec) {
          const uint64_t el = static_cast<uint64_t>(row) * H + vi * 8;
          const uint4 rnd = rng.draw8(el >> 3);
#pragma unroll
          for (int e = 0; e < 8; ++e)
            dv[i][e] = (rand16_of(rnd, e) < rng.thr16) ? 0.f : dv[i][e] * rng.inv_keep;
        }
      }
    }
    const bool active = (p.row_kind == nullptr) || (p.row_kind[row] == p.kind);
    const int nrow = row + stride;   // prefetch the next row of this warp
    if (nrow < p.rows) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int vi = lane + i * 32;
        if (vi < nvec) {
          nx[i] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.x) +
                                                       static_cast<size_t>(nrow) * H) + vi);
          nd[i] = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.dy) +
                                                       static_cast<size_t>(nrow) * H) + vi);
        }
      }
    }
    if (!active) {                   // row belongs to the other LayerNorm (embedding front-end)
      if (p.zero_inactive) {
        uint4* zr = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.dx) + static_cast<size_t>(row) * H);
#pragma unroll
        for (int i = 0; i < NV; ++i)
          if (lane + i * 32 < nvec) zr[lane + i * 32] = make_uint4(0, 0, 0, 0);
      }
      continue;
    }
    const float mean = warp_sum(sum) * inv_h;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + i * 32 < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float d = xv[i][e] - mean; sq += d * d; }
      }
    const float rstd = rsqrtf(warp_sum(sq) * inv_h + LN_EPS);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + i * 32 < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float xh = (xv[i][e] - mean) * rstd;
          const float g = dv[i][e] * gam[i][e];
          s1 += g; s2 += g * xh;
          acc_g[i][e] += dv[i][e] * xh;
          acc_b[i][e] += dv[i][e];
          xv[i][e] = xh;           // keep x-hat
          dv[i][e] = g;            // keep dy * gamma
        }
      }
    s1 = warp_sum(s1) * inv_h;
    s2 = warp_sum(s2) * inv_h;
    uint4* dxr = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.dx) + static_cast<size_t>(row) * H);
    uint4* ddr = p.dx_drop ? reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.dx_drop) +
                                                      static_cast<size_t>(row) * H)
                           : nullptr;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = rstd * (dv[i][e] - s1 - xv[i][e] * s2);
        dxr[vi] = pack8<kBF16>(o);
        if (ddr && !p.dy_drop) {
          const uint64_t el = static_cast<uint64_t>(row) * H + vi * 8;
          const uint4 rnd = rng.draw8(el >> 3);
#pragma unroll
          for (int e = 0; e < 8; ++e)
            o[e] = (rand16_of(rnd, e) < rng.thr16) ? 0.f : o[e] * rng.inv_keep;
          ddr[vi] = pack8<kBF16>(o);
        }
        if (p.dbias) {
#pragma unroll
          for (int e = 0; e < 8; ++e)  // what the Linear branch sees after 16-bit rounding
            acc_d[i][e] += Elem<kBF16>::to_f(Elem<kBF16>::from_f(o[e]));
        }
      }
    }
  }

  // CTA reduction over warps, one vector slot at a time, then one atomic per column per CTA
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      red[0][warp][lane * 8 + e] = acc_g[i][e];
      red[1][warp][lane * 8 + e] = acc_b[i][e];
      red[2][warp][lane * 8 + e] = acc_d[i][e];
    }
    __syncthreads();
    // 64 threads x 4 consecutive columns: one 16-byte vector atomic per quantity instead of four
    // scalar ones (one column-sum atomic per 4 columns instead of one per column)
    if (threadIdx.x < 64) {
      const int c4 = threadIdx.x * 4;
      const int col = c4 + i * 256;
      if (col < H) {
        float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f}, d[4] = {0.f, 0.f, 0.f, 0.f};
        for (int w = 0; w < nwarps; ++w) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            a[q] += red[0][w][c4 + q]; b[q] += red[1][w][c4 + q]; d[q] += red[2][w][c4 + q];
          }
        }
        atomicAdd(reinterpret_cast<float4*>(p.dgamma + col), make_float4(a[0], a[1], a[2], a[3]));
        atomicAdd(reinterpret_cast<float4*>(p.dbeta + col), make_float4(b[0], b[1], b[2], b[3]));
        if (p.dbias) atomicAdd(reinterpret_cast<float4*>(p.dbias + col), make_float4(d[0], d[1], d[2], d[3]));
      }
    }
  }
}

// ------------------------------------------------------------------------------ LayerNorm bwd, split form
// The fused kernel above keeps 3 x NV x 8 column accumulators per thread (240 registers at H = 768:
// one CTA of 8 warps per SM) and every warp walks through a serial chain of 3 warp reductions per
// row, so it runs far below the HBM roofline.  Split form, for the plain case
// (no row-kind mask, dropout on the Linear branch):
//   ln_bwd_rows_kernel  one warp per row, nothing carried between rows (~90 registers: several CTAs
//                       per SM): dx, the dropout-masked copy, and (mean, rstd) of the row to `stats`;
//   ln_bwd_cols_kernel  dgamma / dbeta / dbias as column reductions over a [64 columns x row slab]
//                       block per CTA (the operands are L2-hot), 12x fewer atomics per address.
// kRelu: x is the pre-activation `pre` of y = LN(relu(pre)); xhat comes from relu(pre) and dx_drop
// receives dpre = dx o (pre > 0) (plain rows only: no dropout, no row kind).  Rows wider than 1024
// (NV > 4) keep 16 x NV floats per thread and run one CTA per SM.
template <bool kBF16, int NV, bool kRelu = false>
__global__ void __launch_bounds__(256, NV > 4 ? 1 : 2)
ln_bwd_rows_kernel(const LnBwdParams p, float2* __restrict__ stats) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + warp;
  if (row >= p.rows) return;
  const int H = p.H, nvec = H >> 3;
  const float inv_h = 1.0f / H;
  if (p.row_kind != nullptr && p.row_kind[row] != p.kind) {   // deterministic mode only
    if (p.zero_inactive) {
      uint4* zr = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.dx) + static_cast<size_t>(row) * H);
      for (int vi = lane; vi < nvec; vi += 32) zr[vi] = make_uint4(0, 0, 0, 0);
    }
    return;
  }
  DropoutRng rng;
  rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = p.stream_lo; rng.s1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rng.s0, rng.s1);
  rng.thr16 = p.drop_thr16; rng.inv_keep = p.drop_inv_keep;
  float xv[NV][8], dv[NV][8];
  uint32_t live[kRelu ? NV : 1];   // kRelu: bit e of live[i] = (pre > 0) for column 8 * vi + e
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.x) +
                                                          static_cast<size_t>(row) * H) + vi), xv[i]);
      unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.dy) +
                                                          static_cast<size_t>(row) * H) + vi), dv[i]);
      if constexpr (kRelu) {
        live[i] = 0u;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (xv[i][e] > 0.f) live[i] |= 1u << e;
          else xv[i][e] = 0.f;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) sum += xv[i][e];
      if (p.dy_drop) {               // y = dropout(LN(x)) (deterministic mode only): mask dy
        const uint4 rnd = rng.draw8((static_cast<uint64_t>(row) * H + vi * 8) >> 3);
#pragma unroll
        for (int e = 0; e < 8; ++e) dv[i][e] = (rand16_of(rnd, e) < rng.thr16) ? 0.f : dv[i][e] * rng.inv_keep;
      }
    }
  }
  const float mean = warp_sum(sum) * inv_h;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) { const float d = xv[i][e] - mean; sq += d * d; }
    }
  const float rstd = rsqrtf(warp_sum(sq) * inv_h + LN_EPS);
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float gam[8];
      unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.gamma) + vi), gam);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float xh = (xv[i][e] - mean) * rstd;
        const float g = dv[i][e] * gam[e];
        s1 += g; s2 += g * xh;
        xv[i][e] = xh;
        dv[i][e] = g;
      }
    }
  }
  s1 = warp_sum(s1) * inv_h;
  s2 = warp_sum(s2) * inv_h;
  if (lane == 0) stats[row] = make_float2(mean, rstd);
  uint4* dxr = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.dx) + static_cast<size_t>(row) * H);
  uint4* ddr = p.dx_drop ? reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.dx_drop) + static_cast<size_t>(row) * H)
                         : nullptr;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = rstd * (dv[i][e] - s1 - xv[i][e] * s2);
      dxr[vi] = pack8<kBF16>(o);
      if constexpr (kRelu) {
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = ((live[i] >> e) & 1u) ? o[e] : 0.f;
        ddr[vi] = pack8<kBF16>(o);
      } else if (ddr) {
        const uint64_t el = static_cast<uint64_t>(row) * H + vi * 8;
        const uint4 rnd = rng.draw8(el >> 3);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = (rand16_of(rnd, e) < rng.thr16) ? 0.f : o[e] * rng.inv_keep;
        ddr[vi] = pack8<kBF16>(o);
      }
    }
  }
}

// CTA = 8 column vectors (64 columns) x 32 row lanes over rows [r0, r1).  kRelu: xhat from relu(x).
template <bool kBF16, bool kRelu = false>
__global__ void __launch_bounds__(256)
ln_bwd_cols_kernel(const LnBwdParams p, const float2* __restrict__ stats, int rows_per_cta) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  __shared__ float red[3][32][64 + 1];
  const int cv = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int col0 = (blockIdx.x * 8 + cv) * 8;
  const int r0 = blockIdx.y * rows_per_cta;
  const int r1 = min(p.rows, r0 + rows_per_cta);
  const int H = p.H;
  const void* lin = p.dx_drop ? p.dx_drop : p.dx;      // what the Linear branch receives
  float ag[8], ab[8], ad[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { ag[e] = 0.f; ab[e] = 0.f; ad[e] = 0.f; }
  if (col0 < H) {
    for (int r = r0 + rl; r < r1; r += 32) {
      const float2 st = __ldg(stats + r);
      float x[8], dy[8];
      unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.x) +
                                                          static_cast<size_t>(r) * H + col0)), x);
      unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.dy) +
                                                          static_cast<size_t>(r) * H + col0)), dy);
      if constexpr (kRelu) {
#pragma unroll
        for (int e = 0; e < 8; ++e) x[e] = x[e] > 0.f ? x[e] : 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        ag[e] = fmaf(dy[e], (x[e] - st.x) * st.y, ag[e]);
        ab[e] += dy[e];
      }
      if (p.dbias) {
        float d[8];
        unpack8<kBF16>(*reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(lin) +
                                                       static_cast<size_t>(r) * H + col0), d);
#pragma unroll
        for (int e = 0; e < 8; ++e) ad[e] += d[e];
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    red[0][rl][cv * 8 + e] = ag[e];
    red[1][rl][cv * 8 + e] = ab[e];
    red[2][rl][cv * 8 + e] = ad[e];
  }
  __syncthreads();
  if (threadIdx.x < 192) {
    const int q = threadIdx.x >> 6, c = threadIdx.x & 63;
    const int col = blockIdx.x * 64 + c;
    if (col < H && (q < 2 || p.dbias)) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < 32; ++w) s += red[q][w][c];
      float* dst = q == 0 ? p.dgamma : (q == 1 ? p.dbeta : p.dbias);
      atomicAdd(dst + col, s);
    }
  }
}

// Deterministic form of ln_bwd_cols_kernel: CTA = 8 columns x 256 row lanes over ALL rows, so every
// column has one owner and a fixed summation order (det_tree_sum8).  Also covers the row-kind and
// dropout-on-dy cases of the embedding front-end (the fused kernel's job in the default mode).
// kRelu: xhat from relu(x), as ln_bwd_cols_kernel.
template <bool kBF16, bool kRelu = false>
__global__ void __launch_bounds__(256, 1)   // (256) alone: ptxas caps it at 64 registers and spills
ln_bwd_cols_det_kernel(const LnBwdParams p, const float2* __restrict__ stats) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  __shared__ float red[256][9];
  const int col0 = blockIdx.x * 8;
  const int H = p.H;
  const void* lin = p.dx_drop ? p.dx_drop : p.dx;
  DropoutRng rng;
  rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = p.stream_lo; rng.s1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rng.s0, rng.s1);
  rng.thr16 = p.drop_thr16; rng.inv_keep = p.drop_inv_keep;
  float ag[8], ab[8], ad[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { ag[e] = 0.f; ab[e] = 0.f; ad[e] = 0.f; }
  for (int r = threadIdx.x; r < p.rows; r += 256) {
    if (p.row_kind != nullptr && p.row_kind[r] != p.kind) continue;
    const float2 st = __ldg(stats + r);
    float x[8], dy[8];
    const size_t off = static_cast<size_t>(r) * H + col0;
    unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.x) + off)), x);
    unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.dy) + off)), dy);
    if (p.dy_drop) {
      const uint4 rnd = rng.draw8(off >> 3);
#pragma unroll
      for (int e = 0; e < 8; ++e) dy[e] = (rand16_of(rnd, e) < rng.thr16) ? 0.f : dy[e] * rng.inv_keep;
    }
    if constexpr (kRelu) {
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] = x[e] > 0.f ? x[e] : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      ag[e] = fmaf(dy[e], (x[e] - st.x) * st.y, ag[e]);
      ab[e] += dy[e];
    }
    if (p.dbias) {
      float d[8];
      unpack8<kBF16>(*reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(lin) + off), d);
#pragma unroll
      for (int e = 0; e < 8; ++e) ad[e] += d[e];
    }
  }
  const float sg = det_tree_sum8(ag, red);
  const float sb = det_tree_sum8(ab, red);
  const float sd = det_tree_sum8(ad, red);
  if (threadIdx.x < 8) {
    p.dgamma[col0 + threadIdx.x] += sg;
    p.dbeta[col0 + threadIdx.x] += sb;
    if (p.dbias) p.dbias[col0 + threadIdx.x] += sd;
  }
}

// ------------------------------------------------------------------------------ gather rows
template <int kDummy>
__global__ void __launch_bounds__(256)
gather_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst,
                   const int* __restrict__ idx, int rows, int vec_per_row) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + warp;
  if (row >= rows) return;
  const int s = idx[row];
  uint4* d = dst + static_cast<size_t>(row) * vec_per_row;
  if (s >= 0) {
    const uint4* sp = src + static_cast<size_t>(s) * vec_per_row;
    for (int v = lane; v < vec_per_row; v += 32) d[v] = __ldg(sp + v);
  } else {
    for (int v = lane; v < vec_per_row; v += 32) d[v] = make_uint4(0, 0, 0, 0);
  }
}

// ------------------------------------------------------------------------------ column sum
template <bool kBF16>
__global__ void __launch_bounds__(256)
colsum_kernel(const void* __restrict__ x_, float* __restrict__ out, int rows, int N, int ld,
              int rows_per_cta) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  // CTA = 32 column-vectors (256 columns) x 8 row lanes
  __shared__ float red[8][256 + 1];
  const int cv = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col0 = (blockIdx.x * 32 + cv) * 8;
  const int r0 = blockIdx.y * rows_per_cta;
  const int r1 = min(rows, r0 + rows_per_cta);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col0 < N) {
    for (int r = r0 + rl; r < r1; r += 8) {
      float f[8];
      unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(x_) +
                                                          static_cast<size_t>(r) * ld + col0)), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] += f[e];
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[rl][cv * 8 + e] = acc[e];
  __syncthreads();
  if (threadIdx.x < 64) {            // 4 consecutive columns per thread: one vector atomic
    const int c4 = threadIdx.x * 4;
    const int col = blockIdx.x * 256 + c4;
    if (col < N) {
      float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int w = 0; w < 8; ++w)
#pragma unroll
        for (int q = 0; q < 4; ++q) s[q] += red[w][c4 + q];
      atomicAdd(reinterpret_cast<float4*>(out + col), make_float4(s[0], s[1], s[2], s[3]));
    }
  }
}

// Deterministic column sum: CTA = 8 columns x 256 row lanes over all rows (see det_tree_sum8).
template <bool kBF16>
__global__ void __launch_bounds__(256)
colsum_det_kernel(const void* __restrict__ x_, float* __restrict__ out, int rows, long long ld,
                  const int* __restrict__ rows_dev) {
  pdl_launch_dependents();
  pdl_wait();
  if (rows_dev != nullptr) rows = min(rows, *rows_dev);
  using T16 = typename Elem<kBF16>::T;
  __shared__ float red[256][9];
  const int col0 = blockIdx.x * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int r = threadIdx.x; r < rows; r += 256) {
    float f[8];
    unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(x_) +
                                                        static_cast<size_t>(r) * ld + col0)), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += f[e];
  }
  const float s = det_tree_sum8(acc, red);
  if (threadIdx.x < 8) out[col0 + threadIdx.x] += s;
}

// ------------------------------------------------------------------------------ fp32 -> 16-bit
template <bool kBF16>
__global__ void __launch_bounds__(256)
cvt_kernel(const float* __restrict__ src, void* __restrict__ dst_, long long n, long long nseg,
           long long src_stride, long long dst_stride, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  T16* dst = reinterpret_cast<T16*>(dst_);
  const long long total = n * nseg;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long seg = i / n, j = i - seg * n;
    float v = src[seg * src_stride + j];
    T16* d = dst + seg * dst_stride + j;
    if (accumulate) v += Elem<kBF16>::to_f(*d);
    *d = Elem<kBF16>::from_f(v);
  }
}

// ------------------------------------------------------------------------------ dst = a + b
template <bool kBF16>
__global__ void __launch_bounds__(256)
add16_kernel(uint4* __restrict__ dst, const uint4* __restrict__ a, const uint4* __restrict__ b,
             long long nvec) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float x[8], y[8];
    unpack8<kBF16>(a[i], x);
    unpack8<kBF16>(__ldg(b + i), y);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] += y[e];
    dst[i] = pack8<kBF16>(x);
  }
}

// ------------------------------------------------------------------------------ launchers
template <bool kBF16, bool kRelu>
static cudaError_t launch_ln_fwd_nv(const void* x, const void* gamma, const void* beta, void* y, int rows,
                                    int H, int grid, cudaStream_t stream) {
  switch (ln_wide_nv(H)) {
    case 4: return launch_pdl(ln_fwd_kernel<kBF16, 4, kRelu>, dim3(grid), dim3(256), 0, stream, 1, x, gamma, beta, y, rows, H);
    case 6: return launch_pdl(ln_fwd_kernel<kBF16, 6, kRelu>, dim3(grid), dim3(256), 0, stream, 1, x, gamma, beta, y, rows, H);
    default: return launch_pdl(ln_fwd_kernel<kBF16, 8, kRelu>, dim3(grid), dim3(256), 0, stream, 1, x, gamma, beta, y, rows, H);
  }
}

int launch_ln_fwd(int dtype, const void* x, const void* gamma, const void* beta, void* y, int rows,
                  int H, bool relu, cudaStream_t stream) {
  if (H % 8 != 0 || H > LN_WIDE_MAX_VEC * 256 || rows <= 0)
    return set_error(UB200_EUNSUPPORTED, "ln_fwd: need rows > 0, H %% 8 == 0 and H <= %d (H=%d)",
                     LN_WIDE_MAX_VEC * 256, H);
  const int grid = (rows + 7) / 8;
  ProfScope ps(stream);
  const bool bf = dtype == UB200_BF16;
  if (relu) {
    if (bf) UB_CHECK_CUDA((launch_ln_fwd_nv<true, true>(x, gamma, beta, y, rows, H, grid, stream)));
    else UB_CHECK_CUDA((launch_ln_fwd_nv<false, true>(x, gamma, beta, y, rows, H, grid, stream)));
  } else {
    if (bf) UB_CHECK_CUDA((launch_ln_fwd_nv<true, false>(x, gamma, beta, y, rows, H, grid, stream)));
    else UB_CHECK_CUDA((launch_ln_fwd_nv<false, false>(x, gamma, beta, y, rows, H, grid, stream)));
  }
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

template <bool kBF16>
static cudaError_t launch_ln_bwd_nv(const LnBwdParams& p, int grid, cudaStream_t stream) {
  const int nv = (p.H + 255) / 256;
  switch (nv) {
    case 1: return launch_pdl(ln_bwd_kernel<kBF16, 1>, dim3(grid), dim3(256), 0, stream, 1, p);
    case 2: return launch_pdl(ln_bwd_kernel<kBF16, 2>, dim3(grid), dim3(256), 0, stream, 1, p);
    case 3: return launch_pdl(ln_bwd_kernel<kBF16, 3>, dim3(grid), dim3(256), 0, stream, 1, p);
    default: return launch_pdl(ln_bwd_kernel<kBF16, 4>, dim3(grid), dim3(256), 0, stream, 1, p);
  }
}

template <bool kBF16>
static cudaError_t launch_ln_bwd_rows_nv(const LnBwdParams& p, bool relu, float2* stats, int grid,
                                         cudaStream_t stream) {
  if (relu) {
    switch (ln_wide_nv(p.H)) {
      case 4: return launch_pdl(ln_bwd_rows_kernel<kBF16, 4, true>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
      case 6: return launch_pdl(ln_bwd_rows_kernel<kBF16, 6, true>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
      default: return launch_pdl(ln_bwd_rows_kernel<kBF16, 8, true>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
    }
  }
  const int nv = (p.H + 255) / 256;
  switch (nv) {
    case 1: return launch_pdl(ln_bwd_rows_kernel<kBF16, 1>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
    case 2: return launch_pdl(ln_bwd_rows_kernel<kBF16, 2>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
    case 3: return launch_pdl(ln_bwd_rows_kernel<kBF16, 3>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
    case 4: return launch_pdl(ln_bwd_rows_kernel<kBF16, 4>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
    case 5:
    case 6: return launch_pdl(ln_bwd_rows_kernel<kBF16, 6>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
    default: return launch_pdl(ln_bwd_rows_kernel<kBF16, 8>, dim3(grid), dim3(256), 0, stream, 1, p, stats);
  }
}

template <bool kBF16, bool kRelu>
static cudaError_t launch_ln_bwd_cols(const LnBwdParams& p, const float2* stats, cudaStream_t stream) {
  if (deterministic())
    return launch_pdl(ln_bwd_cols_det_kernel<kBF16, kRelu>, dim3(p.H / 8), dim3(256), 0, stream, 1, p, stats);
  const int gx = (p.H + 63) / 64;
  int gy = (2 * num_sms() + gx - 1) / gx;
  if (gy > (p.rows + 31) / 32) gy = (p.rows + 31) / 32;
  if (gy < 1) gy = 1;
  const int rpc = (p.rows + gy - 1) / gy;
  return launch_pdl(ln_bwd_cols_kernel<kBF16, kRelu>, dim3(gx, gy), dim3(256), 0, stream, 1, p, stats, rpc);
}

// split form (see ln_bwd_rows_kernel): needs `stats` = rows x 2 floats of caller-owned scratch
int launch_ln_bwd_split(int dtype, const LnBwdParams& p, bool relu, float* stats_ws, cudaStream_t stream) {
  float2* stats = reinterpret_cast<float2*>(stats_ws);
  const bool bf = dtype == UB200_BF16;
  {
    ProfScope ps(stream);
    const int grid = (p.rows + 7) / 8;
    if (bf) UB_CHECK_CUDA(launch_ln_bwd_rows_nv<true>(p, relu, stats, grid, stream));
    else UB_CHECK_CUDA(launch_ln_bwd_rows_nv<false>(p, relu, stats, grid, stream));
  }
  ProfScope ps(stream);
  const float2* st = stats;
  if (bf) UB_CHECK_CUDA(relu ? (launch_ln_bwd_cols<true, true>(p, st, stream)) : (launch_ln_bwd_cols<true, false>(p, st, stream)));
  else UB_CHECK_CUDA(relu ? (launch_ln_bwd_cols<false, true>(p, st, stream)) : (launch_ln_bwd_cols<false, false>(p, st, stream)));
  return 0;
}

int launch_ln_bwd(int dtype, const LnBwdParams& p, cudaStream_t stream) {
  if (p.H % 8 != 0 || p.H > LN_MAX_VEC * 256 || p.rows <= 0)
    return set_error(UB200_EUNSUPPORTED, "ln_bwd: need rows > 0, H %% 8 == 0 and H <= %d (H=%d)",
                     LN_MAX_VEC * 256, p.H);
  int grid = (p.rows + 7) / 8;
  const int cap = num_sms();   // one wave
  if (grid > cap) grid = cap;
  ProfScope ps(stream);
  if (dtype == UB200_BF16) UB_CHECK_CUDA(launch_ln_bwd_nv<true>(p, grid, stream));
  else UB_CHECK_CUDA(launch_ln_bwd_nv<false>(p, grid, stream));
  return 0;
}

int launch_gather_rows(const void* src, void* dst, const int* idx, int rows, int row_bytes,
                       cudaStream_t stream) {
  if (row_bytes % 16 != 0 || rows <= 0)
    return set_error(UB200_EINVAL, "gather_rows: rows > 0 and row_bytes %% 16 == 0 required");
  ProfScope ps(stream);
  gather_rows_kernel<0><<<(rows + 7) / 8, 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), idx, rows, row_bytes / 16);
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_colsum_det(int dtype, const void* x, float* out, int rows, int N, long long ld, cudaStream_t stream,
                      const int* rows_dev) {
  if (N % 8 != 0 || ld % 8 != 0 || rows <= 0)
    return set_error(UB200_EINVAL, "colsum: rows > 0, N %% 8 == 0, ld %% 8 == 0 required");
  ProfScope ps(stream);
  if (dtype == UB200_BF16) UB_CHECK_CUDA(launch_pdl(colsum_det_kernel<true>, dim3(N / 8), dim3(256), 0, stream, 1, x, out, rows, ld, rows_dev));
  else UB_CHECK_CUDA(launch_pdl(colsum_det_kernel<false>, dim3(N / 8), dim3(256), 0, stream, 1, x, out, rows, ld, rows_dev));
  return 0;
}

int launch_colsum(int dtype, const void* x, float* out, int rows, int N, int ld, cudaStream_t stream) {
  if (N % 8 != 0 || ld % 8 != 0 || rows <= 0)
    return set_error(UB200_EINVAL, "colsum: rows > 0, N %% 8 == 0, ld %% 8 == 0 required");
  if (deterministic()) return launch_colsum_det(dtype, x, out, rows, N, ld, stream);
  const int gx = (N + 255) / 256;
  int gy = (2 * num_sms() + gx - 1) / gx;
  if (gy > (rows + 31) / 32) gy = (rows + 31) / 32;
  if (gy < 1) gy = 1;
  const int rpc = (rows + gy - 1) / gy;
  dim3 grid(gx, gy);
  ProfScope ps(stream);
  if (dtype == UB200_BF16) UB_CHECK_CUDA(launch_pdl(colsum_kernel<true>, grid, dim3(256), 0, stream, 1, x, out, rows, N, ld, rpc));
  else UB_CHECK_CUDA(launch_pdl(colsum_kernel<false>, grid, dim3(256), 0, stream, 1, x, out, rows, N, ld, rpc));
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_cvt(int dtype, const float* src, void* dst, long long n, long long nseg,
               long long src_stride, long long dst_stride, int accumulate, cudaStream_t stream) {
  if (n <= 0 || nseg <= 0) return 0;
  long long blocks = (n * nseg + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  ProfScope ps(stream);
  if (dtype == UB200_BF16)
    UB_CHECK_CUDA(launch_pdl(cvt_kernel<true>, dim3(static_cast<int>(blocks)), dim3(256), 0, stream, 1, src, dst, n, nseg, src_stride, dst_stride, accumulate));
  else
    UB_CHECK_CUDA(launch_pdl(cvt_kernel<false>, dim3(static_cast<int>(blocks)), dim3(256), 0, stream, 1, src, dst, n, nseg, src_stride, dst_stride, accumulate));
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int launch_add16(int dtype, void* dst, const void* a, const void* b, long long n, cudaStream_t stream) {
  if (n % 8 != 0) return set_error(UB200_EINVAL, "add16: n %% 8 != 0");
  const long long nvec = n / 8;
  long long blocks = (nvec + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  ProfScope ps(stream);
  if (dtype == UB200_BF16)
    add16_kernel<true><<<static_cast<int>(blocks), 256, 0, stream>>>(
        reinterpret_cast<uint4*>(dst), reinterpret_cast<const uint4*>(a),
        reinterpret_cast<const uint4*>(b), nvec);
  else
    add16_kernel<false><<<static_cast<int>(blocks), 256, 0, stream>>>(
        reinterpret_cast<uint4*>(dst), reinterpret_cast<const uint4*>(a),
        reinterpret_cast<const uint4*>(b), nvec);
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ub

// ------------------------------------------------------------------------------ C ABI
extern "C" int ub200_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y,
                                   int32_t rows, int32_t hidden, int32_t dtype,
                                   ub200_stream_t stream) {
  UB_CHECK_ARG(x && gamma && beta && y, "layernorm_fwd: null pointer");
  return ub::launch_ln_fwd(dtype, x, gamma, beta, y, rows, hidden, false,
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ub200_layernorm_fwd_act(const void* x, const void* gamma, const void* beta, void* y,
                                       int32_t rows, int32_t hidden, int32_t dtype, int32_t act,
                                       ub200_stream_t stream) {
  UB_CHECK_ARG(x && gamma && beta && y, "layernorm_fwd_act: null pointer");
  UB_CHECK_ARG(act == UB200_LN_ACT_NONE || act == UB200_LN_ACT_RELU, "layernorm_fwd_act: unknown act %d", act);
  return ub::launch_ln_fwd(dtype, x, gamma, beta, y, rows, hidden, act == UB200_LN_ACT_RELU,
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ub200_layernorm_bwd(const ub200_ln_bwd_args* a, ub200_stream_t stream) {
  UB_CHECK_ARG(a && a->dy && a->x && a->gamma && a->dx && a->dgamma && a->dbeta,
               "layernorm_bwd: null pointer");
  UB_CHECK_ARG(((reinterpret_cast<uintptr_t>(a->dgamma) | reinterpret_cast<uintptr_t>(a->dbeta) |
                 reinterpret_cast<uintptr_t>(a->dbias)) & 15) == 0,
               "layernorm_bwd: dgamma / dbeta / dbias must be 16-byte aligned (vector atomics)");
  ub::LnBwdParams p{};
  p.dy = a->dy; p.x = a->x; p.gamma = a->gamma; p.dx = a->dx;
  p.dgamma = a->dgamma; p.dbeta = a->dbeta; p.dbias = a->dbias;
  p.rows = a->rows; p.H = a->hidden;
  p.row_kind = a->row_kind; p.kind = a->kind; p.dy_drop = 0;
  p.zero_inactive = (a->dropout_on_dy & 2) ? 1 : 0;
  if (a->dropout_p > 0.f) {
    UB_CHECK_ARG(a->dx_drop || (a->dropout_on_dy & 1), "layernorm_bwd: dropout_p > 0 needs dx_drop");
    const ub::DropoutThreshold d = ub::dropout_threshold(a->dropout_p);
    p.dx_drop = (a->dropout_on_dy & 1) ? nullptr : a->dx_drop;
    p.dy_drop = (a->dropout_on_dy & 1) ? 1 : 0;
    p.drop_thr16 = d.thr16;
    p.drop_inv_keep = d.inv_keep;
  } else {
    p.dx_drop = nullptr; p.drop_thr16 = 0; p.drop_inv_keep = 1.f;
  }
  p.seed_lo = static_cast<uint32_t>(a->rng_seed); p.seed_hi = static_cast<uint32_t>(a->rng_seed >> 32);
  p.stream_lo = static_cast<uint32_t>(a->rng_stream);
  p.stream_hi = static_cast<uint32_t>(a->rng_stream >> 32);
  p.rng_dev = reinterpret_cast<const unsigned long long*>(a->rng_offset_dev);
  UB_CHECK_ARG(a->act == UB200_LN_ACT_NONE || a->act == UB200_LN_ACT_RELU, "layernorm_bwd: unknown act %d", a->act);
  const bool relu = a->act == UB200_LN_ACT_RELU;
  // The split form (row kernel + column kernel, fixed-order in the deterministic mode) is the only one
  // for ReLU rows and rows wider than 1024, the deterministic mode takes it for every case, and
  // stats_ws selects it for plain rows (no row_kind, no dropout on dy).
  const bool split_only = relu || p.H > ub::LN_MAX_VEC * 256;
  const bool plain = a->row_kind == nullptr && !p.dy_drop;
  if (!(split_only || ub::deterministic() || (a->stats_ws != nullptr && plain)))
    return ub::launch_ln_bwd(a->dtype, p, reinterpret_cast<cudaStream_t>(stream));
  UB_CHECK_ARG(a->stats_ws != nullptr,
               "layernorm_bwd: ReLU, hidden > %d and the deterministic mode need stats_ws (rows x 2 floats)",
               ub::LN_MAX_VEC * 256);
  UB_CHECK_ARG((reinterpret_cast<uintptr_t>(a->stats_ws) & 7) == 0, "layernorm_bwd: stats_ws must be 8-byte aligned");
  UB_CHECK_ARG(!split_only || (a->row_kind == nullptr && !(a->dropout_on_dy & 1)),
               "layernorm_bwd: ReLU or hidden > %d takes no row_kind and no dropout on dy", ub::LN_MAX_VEC * 256);
  if (relu) {   // dx_drop receives dpre = dx o (pre > 0)
    UB_CHECK_ARG(a->dx_drop != nullptr, "layernorm_bwd: ReLU needs dx_drop (it receives dpre)");
    UB_CHECK_ARG(a->dropout_p == 0.f, "layernorm_bwd: ReLU and dropout share dx_drop; dropout_p must be 0");
    p.dx_drop = a->dx_drop;
  }
  if (p.H % 8 != 0 || p.H > ub::LN_WIDE_MAX_VEC * 256 || p.rows <= 0)
    return ub::set_error(UB200_EUNSUPPORTED, "ln_bwd: need rows > 0, H %% 8 == 0 and H <= %d (H=%d)",
                         ub::LN_WIDE_MAX_VEC * 256, p.H);
  return ub::launch_ln_bwd_split(a->dtype, p, relu, a->stats_ws, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ub200_gather_rows(const void* src, void* dst, const int32_t* index, int32_t rows,
                                 int32_t row_bytes, ub200_stream_t stream) {
  UB_CHECK_ARG(src && dst && index, "gather_rows: null pointer");
  return ub::launch_gather_rows(src, dst, index, rows, row_bytes,
                                reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ub200_colsum(const void* x, float* out, int32_t rows, int32_t cols, int64_t ld,
                            int32_t dtype, ub200_stream_t stream) {
  UB_CHECK_ARG(x && out, "colsum: null pointer");
  UB_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15) == 0, "colsum: out must be 16-byte aligned (vector atomics)");
  return ub::launch_colsum(dtype, x, out, rows, cols, static_cast<int>(ld),
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ub200_cvt_from_f32(const float* src, void* dst, int64_t n, int32_t accumulate,
                                  int32_t dtype, ub200_stream_t stream) {
  UB_CHECK_ARG(src && dst, "cvt_from_f32: null pointer");
  return ub::launch_cvt(dtype, src, dst, n, 1, 0, 0, accumulate, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int ub200_cvt_from_f32_strided(const float* src, void* dst, int64_t n, int64_t nseg,
                                          int64_t src_stride, int64_t dst_stride, int32_t accumulate,
                                          int32_t dtype, ub200_stream_t stream) {
  UB_CHECK_ARG(src && dst, "cvt_from_f32_strided: null pointer");
  UB_CHECK_ARG(n >= 0 && nseg >= 0, "cvt_from_f32_strided: negative size");
  return ub::launch_cvt(dtype, src, dst, n, nseg, src_stride, dst_stride, accumulate,
                        reinterpret_cast<cudaStream_t>(stream));
}
