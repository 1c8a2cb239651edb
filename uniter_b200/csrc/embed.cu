// Embedding front-end of UniterModel, computed straight into PACKED rows.
//
// Reference (model/model.py): UniterTextEmbeddings.forward :232-245 (3 gathers + add + LN +
// dropout), UniterImageEmbeddings.forward :261-272 (+mask embedding, img_linear, 3 LayerNorms,
// pos_linear with K = 7, dropout), _compute_img_txt_embeddings :321-334 (cat + torch.gather with
// gather_index).  The reference materialises [B, Lt, H], [B, Li, H], their concatenation and the
// gathered [B, L, H]; here packed row t is produced directly from its source row
//     src = gather_index[b, j]  (text row if src < Lt, else region src - Lt)
// so padding rows are never computed and an arbitrary gather_index is honoured by construction.
//
//   embed_prep        integer bookkeeping per packed row (bit-exact indexing)
//   embed_gather_cast region features (fp32 or 16-bit) -> 16-bit [T, D] operand of the img_linear
//                     GEMM (+ mask_embedding row for masked regions, zeros for text rows)
//   embed_rows_fwd    one warp per packed row: text  LN(word + pos + type)
//                                              image LN( LN(G) + LN(pos_linear(box)) + type )
//                     + Philox dropout; also saves the two / three pre-LayerNorm sums that the
//                     backward LayerNorm kernels need.
// Backward = ub200_layernorm_bwd (row-kind masked) + wgrad GEMM + table scatter (host side).
#include "common.h"
#include "ptx.cuh"

namespace ub {

constexpr int EMB_MAX_VEC = 4;   // H <= 1024
constexpr float EMB_EPS = 1e-12f;

template <bool kBF16>
__device__ __forceinline__ void e_unpack8(const uint4& u, float* f) {
  float2 t;
  t = Elem<kBF16>::unpack(u.x); f[0] = t.x; f[1] = t.y;
  t = Elem<kBF16>::unpack(u.y); f[2] = t.x; f[3] = t.y;
  t = Elem<kBF16>::unpack(u.z); f[4] = t.x; f[5] = t.y;
  t = Elem<kBF16>::unpack(u.w); f[6] = t.x; f[7] = t.y;
}
template <bool kBF16>
__device__ __forceinline__ uint4 e_pack8(const float* f) {
  uint4 u;
  u.x = Elem<kBF16>::pack(f[0], f[1]); u.y = Elem<kBF16>::pack(f[2], f[3]);
  u.z = Elem<kBF16>::pack(f[4], f[5]); u.w = Elem<kBF16>::pack(f[6], f[7]);
  return u;
}
__device__ __forceinline__ float e_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------ index prep
struct PrepParams {
  const int* pack_idx;            // [T] -> b * L + j
  const long long* gather_index;  // [B, L] or NULL (text-only / image-only: src = j)
  const long long* input_ids;     // [B, Lt] or NULL
  const long long* position_ids;  // [pos_rows, Lt]
  const long long* txt_type_ids;  // [B, Lt] or NULL (-> 0)
  const long long* img_type_ids;  // [B, Li] or NULL (-> 1)
  const unsigned char* img_masks; // [B, Li] (bool / uint8) or NULL
  int T, L, Lt, Li, pos_rows, mode;  // mode 0 joint, 1 text only, 2 image only
  int* kind; int* word_id; int* pos_id; int* type_id; int* img_src; int* mask_flag;
};

__global__ void embed_prep_kernel(const PrepParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.T) return;
  const int flat = p.pack_idx[t];
  const int b = flat / p.L, j = flat % p.L;
  long long src = (p.mode == 0) ? p.gather_index[flat] : j;
  const bool is_txt = (p.mode == 1) || (p.mode == 0 && src < p.Lt);
  int kind, wid = 0, pid = 0, tid = 0, isrc = -1, mflag = 0;
  if (is_txt) {
    kind = 0;
    const long long o = static_cast<long long>(b) * p.Lt + src;
    wid = static_cast<int>(p.input_ids[o]);
    pid = static_cast<int>(p.position_ids[(p.pos_rows == 1 ? 0 : static_cast<long long>(b) * p.Lt) + src]);
    tid = p.txt_type_ids ? static_cast<int>(p.txt_type_ids[o]) : 0;
  } else {
    kind = 1;
    const long long r = (p.mode == 0) ? src - p.Lt : src;
    const long long o = static_cast<long long>(b) * p.Li + r;
    isrc = static_cast<int>(o);
    tid = p.img_type_ids ? static_cast<int>(p.img_type_ids[o]) : 1;
    mflag = p.img_masks ? (p.img_masks[o] != 0) : 0;
  }
  p.kind[t] = kind; p.word_id[t] = wid; p.pos_id[t] = pid; p.type_id[t] = tid;
  p.img_src[t] = isrc; p.mask_flag[t] = mflag;
}

// ------------------------------------------------------------------------------ gather + cast
// out[t, :] = 16-bit( img_feat[img_src[t], :] (+ mask_row if mask_flag[t]) ), zeros for text rows.
template <bool kBF16, typename TIn>
__global__ void __launch_bounds__(256)
embed_gather_cast_kernel(const TIn* __restrict__ feat, const int* __restrict__ img_src,
                         const int* __restrict__ mask_flag, const void* __restrict__ mask_row_,
                         void* __restrict__ out_, int T, int D) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * (blockDim.x >> 5) + warp;
  if (t >= T) return;
  const int s = img_src[t];
  uint4* out = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(out_) + static_cast<size_t>(t) * D);
  const int nvec = D >> 3;
  if (s < 0) {
    for (int v = lane; v < nvec; v += 32) out[v] = make_uint4(0, 0, 0, 0);
    return;
  }
  const bool add_mask = mask_flag[t] != 0;
  const TIn* src = feat + static_cast<size_t>(s) * D;
  for (int v = lane; v < nvec; v += 32) {
    float f[8];
    if (sizeof(TIn) == 4) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src) + 2 * v);
      const float4 b = __ldg(reinterpret_cast<const float4*>(src) + 2 * v + 1);
      f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    } else {
      e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(src) + v), f);
    }
    if (add_mask) {
      // the reference adds in the model dtype: round the feature first, then add (model.py:264-265)
      float m[8];
      e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(mask_row_) + v), m);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(f[e])) + m[e];
    }
    out[v] = e_pack8<kBF16>(f);
  }
}

// ------------------------------------------------------------------------------ fused rows fwd
struct RowsParams {
  const int* kind; const int* word_id; const int* pos_id; const int* type_id; const int* img_src;
  const void* word_emb; const void* pos_emb; const void* type_emb;   // [V,H] [P,H] [Ty,H] 16-bit
  const void* ln_t_g; const void* ln_t_b;                             // embeddings.LayerNorm
  const void* G;                                                      // [T,H] img_linear output (16-bit)
  const float* pos_feat;                                              // [B*Li, 7] fp32 boxes
  const void* w_pos; const void* b_pos;                               // [H,7], [H] 16-bit
  const void* ln_i_g; const void* ln_i_b;                             // img_layer_norm
  const void* ln_p_g; const void* ln_p_b;                             // pos_layer_norm
  const void* ln_f_g; const void* ln_f_b;                             // img_embeddings.LayerNorm
  void* x;        // [T,H] output (after dropout)
  void* u;        // [T,H] pre-final-LayerNorm sum (saved for backward)
  void* ppre;     // [T,H] pos_linear output, zeros for text rows (saved for backward)
  int T, H;
  uint32_t drop_thr16; float drop_inv_keep;
  uint32_t seed_lo, seed_hi, stream_lo, stream_hi;
  const unsigned long long* rng_dev;   // optional device-side dropout stream offset (graph replay)
};

template <bool kBF16, int NV>
__global__ void __launch_bounds__(256)
embed_rows_fwd_kernel(const RowsParams p) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * (blockDim.x >> 5) + warp;
  if (t >= p.T) return;
  const int H = p.H, nvec = H >> 3;
  const float inv_h = 1.0f / H;
  const int kind = p.kind[t];
  float v[NV][8];
  auto row16 = [&](const void* base, long long row) {
    return reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(base) + row * H);
  };
  // LayerNorm of v in place (fp32 statistics), affine from g / b
  auto layer_norm = [&](const void* g, const void* b) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + i * 32 < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) s += v[i][e];
      }
    const float mean = e_warp_sum(s) * inv_h;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + i * 32 < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float d = v[i][e] - mean; q += d * d; }
      }
    const float rstd = rsqrtf(e_warp_sum(q) * inv_h + EMB_EPS);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float gg[8], bb[8];
        e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(g) + vi), gg);
        e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(b) + vi), bb);
#pragma unroll
        for (int e = 0; e < 8; ++e)   // LayerNorm outputs are 16-bit tensors in the reference
          v[i][e] = Elem<kBF16>::to_f(Elem<kBF16>::from_f((v[i][e] - mean) * rstd * gg[e] + bb[e]));
      }
    }
  };

  uint4* urow = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.u) + static_cast<size_t>(t) * H);
  uint4* prow = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.ppre) + static_cast<size_t>(t) * H);
  const uint4* tyrow = row16(p.type_emb, p.type_id[t]);
  if (kind == 0) {
    const uint4* w = row16(p.word_emb, p.word_id[t]);
    const uint4* ps = row16(p.pos_emb, p.pos_id[t]);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float a[8], b[8], c[8];
        e_unpack8<kBF16>(__ldg(w + vi), a);
        e_unpack8<kBF16>(__ldg(ps + vi), b);
        e_unpack8<kBF16>(__ldg(tyrow + vi), c);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[i][e] = a[e] + b[e] + c[e];
        urow[vi] = e_pack8<kBF16>(v[i]);
        prow[vi] = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[i][e] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(v[i][e]));
      }
    }
    layer_norm(p.ln_t_g, p.ln_t_b);
  } else {
    // ---- LN(pos_linear(box)) : K = 7 contraction per output column
    const float* box = p.pos_feat + static_cast<size_t>(p.img_src[t]) * 7;
    float f7[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) f7[k] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(__ldg(box + k)));
    float pl[NV][8];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float bb[8];
        e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(p.b_pos) + vi), bb);
        const T16* wp = reinterpret_cast<const T16*>(p.w_pos) + static_cast<size_t>(vi) * 8 * 7;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float acc = bb[e];
#pragma unroll
          for (int k = 0; k < 7; ++k) acc = fmaf(Elem<kBF16>::to_f(wp[e * 7 + k]), f7[k], acc);
          v[i][e] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(acc));
        }
        prow[vi] = e_pack8<kBF16>(v[i]);
      }
    }
    layer_norm(p.ln_p_g, p.ln_p_b);
#pragma unroll
    for (int i = 0; i < NV; ++i)
#pragma unroll
      for (int e = 0; e < 8; ++e) pl[i][e] = v[i][e];
    // ---- LN(img_linear(feat))
    const uint4* g = row16(p.G, t);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) e_unpack8<kBF16>(__ldg(g + vi), v[i]);
    }
    layer_norm(p.ln_i_g, p.ln_i_b);
    // ---- sum + type, final LN
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int vi = lane + i * 32;
      if (vi < nvec) {
        float c[8];
        e_unpack8<kBF16>(__ldg(tyrow + vi), c);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[i][e] = v[i][e] + pl[i][e] + c[e];
        urow[vi] = e_pack8<kBF16>(v[i]);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[i][e] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(v[i][e]));
      }
    }
    layer_norm(p.ln_f_g, p.ln_f_b);
  }
  // ---- dropout + store
  DropoutRng rng;
  rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = p.stream_lo; rng.s1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rng.s0, rng.s1);
  uint4* xrow = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(p.x) + static_cast<size_t>(t) * H);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      if (p.drop_thr16) {
        const uint64_t el = static_cast<uint64_t>(t) * H + vi * 8;
        const uint4 rnd = rng.draw8(el >> 3);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          v[i][e] = (rand16_of(rnd, e) < p.drop_thr16) ? 0.f : v[i][e] * p.drop_inv_keep;
      }
      xrow[vi] = e_pack8<kBF16>(v[i]);
    }
  }
}


// ------------------------------------------------------------------------------ backward: tables
// Gradient of the three embedding-table lookups of a TEXT row (model/model.py:235-237):
//   d_word[word_id[t]] += du[t]   16-bit packed atomics into the pre-zeroed [V, H] gradient
//                                 (what torch's index_add_ does in the model dtype)
//   d_pos [pos_id[t]]  += du[t]   fp32 atomics ([P, H] staging, converted once afterwards)
// One warp per packed row, 16-byte loads; image rows return immediately.
template <bool kBF16>
__global__ void __launch_bounds__(256)
embed_bwd_scatter_kernel(const void* __restrict__ du_, const int* __restrict__ kind,
                         const int* __restrict__ word_id, const int* __restrict__ pos_id,
                         void* __restrict__ d_word_, float* __restrict__ d_pos, int T, int H) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  using T16x2 = typename Elem<kBF16>::T2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = blockIdx.x * (blockDim.x >> 5) + warp;
  if (t >= T || kind[t] != 0) return;
  const int nvec = H >> 3;
  const uint4* du = reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(du_) + static_cast<size_t>(t) * H);
  T16* wrow = reinterpret_cast<T16*>(d_word_) + static_cast<size_t>(word_id[t]) * H;
  float* prow = d_pos + static_cast<size_t>(pos_id[t]) * H;
  for (int v = lane; v < nvec; v += 32) {
    const uint4 u = __ldg(du + v);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      T16x2 pr;
      *reinterpret_cast<uint32_t*>(&pr) = w[q];
      atomicAdd(reinterpret_cast<T16x2*>(wrow + v * 8 + q * 2), pr);
      const float2 f = Elem<kBF16>::unpack(w[q]);
      atomicAdd(prow + v * 8 + q * 2, f.x);
      atomicAdd(prow + v * 8 + q * 2 + 1, f.y);
    }
  }
}

// Deterministic form (one CTA of 128 threads per packed row; blockIdx.y = 0 word table, 1 position
// table).  The CTA of the FIRST text row with a given id owns that id: it sums the du rows of every
// text row with the id in ascending row order in fp32 (8 columns per thread) and adds the total to the
// table row once, rounding once as torch's deterministic embedding backward does.  Other rows exit
// after the ownership scan.  Needs hidden <= 1024.
template <bool kBF16>
__global__ void __launch_bounds__(128)
embed_bwd_scatter_det_kernel(const void* __restrict__ du_, const int* __restrict__ kind,
                             const int* __restrict__ word_id, const int* __restrict__ pos_id,
                             void* __restrict__ d_word_, float* __restrict__ d_pos, int T, int H) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  __shared__ unsigned match[4];
  const int t = blockIdx.x;
  if (kind[t] != 0) return;
  const int* ids = blockIdx.y ? pos_id : word_id;
  const int id = ids[t];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  bool earlier = false;
  for (int r = tid; r < t && !earlier; r += 128) earlier = kind[r] == 0 && ids[r] == id;
  if (__syncthreads_or(earlier)) return;
  const int v = tid;                         // this thread's 8 columns
  const bool col_ok = v < (H >> 3);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int base = t; base < T; base += 128) {
    const int r = base + tid;
    const bool m = r < T && kind[r] == 0 && ids[r] == id;
    const unsigned b = __ballot_sync(0xffffffffu, m);
    if (lane == 0) match[warp] = b;
    __syncthreads();
    if (col_ok) {
      for (int w = 0; w < 4; ++w) {
        unsigned bits = match[w];
        while (bits) {
          const int row = base + w * 32 + __ffs(bits) - 1;
          bits &= bits - 1;
          float f[8];
          e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(du_) +
                                                                static_cast<size_t>(row) * H) + v), f);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] += f[e];
        }
      }
    }
    __syncthreads();
  }
  if (!col_ok) return;
  if (blockIdx.y == 0) {
    uint4* w = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(d_word_) + static_cast<size_t>(id) * H) + v;
    float cur[8];
    e_unpack8<kBF16>(*w, cur);
    uint32_t o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) o[q] = Elem<kBF16>::pack(cur[2 * q] + acc[2 * q], cur[2 * q + 1] + acc[2 * q + 1]);
    *w = make_uint4(o[0], o[1], o[2], o[3]);
  } else {
    float* prow = d_pos + static_cast<size_t>(id) * H + v * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) prow[e] += acc[e];
  }
}

// ------------------------------------------------------------------------------ weighted column sums
//   out[k * stride_k + n * stride_n] += sum_t w_k(t) * x[t, n],   k < W
// mode 0  w_k(t) = (type_id[t] - base == k)               -> token_type table gradient [Ty, H]
// mode 1  w_k(t) = 16-bit(pos_feat[img_src[t], k]), k < 7 -> pos_linear.weight gradient [H, 7]
//                  (image rows only: the K = 7 wgrad of model/model.py:258 as a reduction)
// CTA = 32 column vectors (256 columns) x 8 row lanes over a slab of rows; per-thread fp32
// accumulators, one smem reduction and one atomic per (k, column) per CTA.
struct WColsumParams {
  const void* x;            // [T, N] 16-bit
  const int* type_id;       // mode 0
  const int* kind;          // mode 1
  const int* img_src;       // mode 1
  const float* pos_feat;    // mode 1: [*, 7] fp32
  float* out;
  int T, N, mode, base, nweights, rows_per_cta;
  long long stride_k, stride_n;
};

template <bool kBF16>
__global__ void __launch_bounds__(256)
wcolsum_kernel(const WColsumParams p) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  constexpr int W = 8;
  __shared__ float red[8][256 + 1];
  const int cv = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col0 = (blockIdx.x * 32 + cv) * 8;
  const int r0 = blockIdx.y * p.rows_per_cta;
  const int r1 = min(p.T, r0 + p.rows_per_cta);
  float acc[W][8];
#pragma unroll
  for (int k = 0; k < W; ++k)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[k][e] = 0.f;
  if (col0 < p.N) {
    for (int r = r0 + rl; r < r1; r += 8) {
      float w[W];
#pragma unroll
      for (int k = 0; k < W; ++k) w[k] = 0.f;
      bool any = false;
      if (p.mode == 0) {
        const int ty = p.type_id[r] - p.base;
        if (ty >= 0 && ty < W) {
          any = true;
#pragma unroll
          for (int k = 0; k < W; ++k) w[k] = (ty == k) ? 1.f : 0.f;
        }
      } else {
        const int s = p.img_src[r];
        if (p.kind[r] == 1 && s >= 0) {
          any = true;
          const float* box = p.pos_feat + static_cast<size_t>(s) * 7;
#pragma unroll
          for (int k = 0; k < 7; ++k) w[k] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(__ldg(box + k)));
        }
      }
      if (!any) continue;
      float f[8];
      e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.x) +
                                                            static_cast<size_t>(r) * p.N + col0)), f);
#pragma unroll
      for (int k = 0; k < W; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[k][e] = fmaf(w[k], f[e], acc[k][e]);
    }
  }
  const int c = threadIdx.x;
  const int col = blockIdx.x * 256 + c;
#pragma unroll
  for (int k = 0; k < W; ++k) {
    if (k >= p.nweights) break;     // uniform
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 8; ++e) red[rl][cv * 8 + e] = acc[k][e];
    __syncthreads();
    if (col < p.N) {
      float s = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) s += red[w8][c];
      if (s != 0.f) atomicAdd(p.out + k * p.stride_k + col * p.stride_n, s);
    }
  }
}

// Deterministic form: CTA = 8 columns x 256 row lanes over all rows (det_tree_sum8), one owner per output.
template <bool kBF16>
__global__ void __launch_bounds__(256)
wcolsum_det_kernel(const WColsumParams p) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  constexpr int W = 8;
  __shared__ float red[256][9];
  const int col0 = blockIdx.x * 8;
  float acc[W][8];
#pragma unroll
  for (int k = 0; k < W; ++k)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[k][e] = 0.f;
  for (int r = threadIdx.x; r < p.T; r += 256) {
    float w[W];
#pragma unroll
    for (int k = 0; k < W; ++k) w[k] = 0.f;
    if (p.mode == 0) {
      const int ty = p.type_id[r] - p.base;
      if (ty < 0 || ty >= W) continue;
#pragma unroll
      for (int k = 0; k < W; ++k) w[k] = (ty == k) ? 1.f : 0.f;
    } else {
      const int s = p.img_src[r];
      if (p.kind[r] != 1 || s < 0) continue;
      const float* box = p.pos_feat + static_cast<size_t>(s) * 7;
#pragma unroll
      for (int k = 0; k < 7; ++k) w[k] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(__ldg(box + k)));
    }
    float f[8];
    e_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.x) +
                                                          static_cast<size_t>(r) * p.N + col0)), f);
#pragma unroll
    for (int k = 0; k < W; ++k)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[k][e] = fmaf(w[k], f[e], acc[k][e]);
  }
#pragma unroll
  for (int k = 0; k < W; ++k) {
    if (k >= p.nweights) break;     // uniform
    const float s = det_tree_sum8(acc[k], red);
    if (threadIdx.x < 8) p.out[k * p.stride_k + (col0 + threadIdx.x) * p.stride_n] += s;
  }
}

}  // namespace ub

// ------------------------------------------------------------------------------ C ABI
extern "C" int ub200_embed_prep(const ub200_embed_prep_args* a, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(a && a->pack_idx && a->kind && a->word_id && a->pos_id && a->type_id && a->img_src &&
                   a->mask_flag, "embed_prep: null pointer");
  UB_CHECK_ARG(a->T > 0 && a->L > 0, "embed_prep: empty problem");
  UB_CHECK_ARG(a->mode >= 0 && a->mode <= 2, "embed_prep: bad mode %d", a->mode);
  UB_CHECK_ARG(a->mode == 2 || (a->input_ids && a->position_ids && a->Lt > 0),
               "embed_prep: text inputs missing");
  UB_CHECK_ARG(a->mode != 0 || a->gather_index, "embed_prep: joint mode needs gather_index");
  PrepParams p{};
  p.pack_idx = a->pack_idx; p.gather_index = reinterpret_cast<const long long*>(a->gather_index);
  p.input_ids = reinterpret_cast<const long long*>(a->input_ids);
  p.position_ids = reinterpret_cast<const long long*>(a->position_ids);
  p.txt_type_ids = reinterpret_cast<const long long*>(a->txt_type_ids);
  p.img_type_ids = reinterpret_cast<const long long*>(a->img_type_ids);
  p.img_masks = a->img_masks;
  p.T = a->T; p.L = a->L; p.Lt = a->Lt; p.Li = a->Li; p.pos_rows = a->pos_rows; p.mode = a->mode;
  p.kind = a->kind; p.word_id = a->word_id; p.pos_id = a->pos_id; p.type_id = a->type_id;
  p.img_src = a->img_src; p.mask_flag = a->mask_flag;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(stream);
  embed_prep_kernel<<<(a->T + 255) / 256, 256, 0, stream>>>(p);
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int ub200_embed_gather_cast(const void* img_feat, int32_t feat_is_f32, const int32_t* img_src,
                                       const int32_t* mask_flag, const void* mask_row, void* out,
                                       int32_t T, int32_t D, int32_t dtype, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(img_feat && img_src && mask_flag && mask_row && out, "embed_gather_cast: null pointer");
  UB_CHECK_ARG(T > 0 && D > 0 && D % 8 == 0, "embed_gather_cast: need T > 0 and D %% 8 == 0");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int grid = (T + 7) / 8;
  ProfScope ps(stream);
  if (dtype == UB200_BF16) {
    if (feat_is_f32)
      embed_gather_cast_kernel<true, float><<<grid, 256, 0, stream>>>(
          reinterpret_cast<const float*>(img_feat), img_src, mask_flag, mask_row, out, T, D);
    else
      embed_gather_cast_kernel<true, __nv_bfloat16><<<grid, 256, 0, stream>>>(
          reinterpret_cast<const __nv_bfloat16*>(img_feat), img_src, mask_flag, mask_row, out, T, D);
  } else {
    if (feat_is_f32)
      embed_gather_cast_kernel<false, float><<<grid, 256, 0, stream>>>(
          reinterpret_cast<const float*>(img_feat), img_src, mask_flag, mask_row, out, T, D);
    else
      embed_gather_cast_kernel<false, __half><<<grid, 256, 0, stream>>>(
          reinterpret_cast<const __half*>(img_feat), img_src, mask_flag, mask_row, out, T, D);
  }
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int ub200_embed_rows_fwd(const ub200_embed_rows_args* a, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(a && a->kind && a->word_id && a->pos_id && a->type_id && a->img_src && a->type_emb &&
                   a->x && a->u && a->ppre, "embed_rows_fwd: null pointer");
  UB_CHECK_ARG(a->T > 0 && a->hidden > 0 && a->hidden % 8 == 0 && a->hidden <= EMB_MAX_VEC * 256,
               "embed_rows_fwd: need T > 0, hidden %% 8 == 0, hidden <= %d", EMB_MAX_VEC * 256);
  UB_CHECK_ARG(a->dropout_p >= 0.f && a->dropout_p < 1.f, "embed_rows_fwd: dropout_p out of range");
  RowsParams p{};
  p.kind = a->kind; p.word_id = a->word_id; p.pos_id = a->pos_id; p.type_id = a->type_id;
  p.img_src = a->img_src;
  p.word_emb = a->word_emb; p.pos_emb = a->pos_emb; p.type_emb = a->type_emb;
  p.ln_t_g = a->ln_txt_g; p.ln_t_b = a->ln_txt_b;
  p.G = a->img_linear_out; p.pos_feat = a->pos_feat; p.w_pos = a->w_pos; p.b_pos = a->b_pos;
  p.ln_i_g = a->ln_img_g; p.ln_i_b = a->ln_img_b; p.ln_p_g = a->ln_pos_g; p.ln_p_b = a->ln_pos_b;
  p.ln_f_g = a->ln_out_g; p.ln_f_b = a->ln_out_b;
  p.x = a->x; p.u = a->u; p.ppre = a->ppre; p.T = a->T; p.H = a->hidden;
  if (a->dropout_p > 0.f) {
    const DropoutThreshold d = dropout_threshold(a->dropout_p);
    p.drop_thr16 = d.thr16; p.drop_inv_keep = d.inv_keep;
  } else {
    p.drop_thr16 = 0; p.drop_inv_keep = 1.f;
  }
  p.seed_lo = static_cast<uint32_t>(a->rng_seed); p.seed_hi = static_cast<uint32_t>(a->rng_seed >> 32);
  p.stream_lo = static_cast<uint32_t>(a->rng_stream); p.stream_hi = static_cast<uint32_t>(a->rng_stream >> 32);
  p.rng_dev = reinterpret_cast<const unsigned long long*>(a->rng_offset_dev);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int grid = (a->T + 7) / 8;
  const int nv = (a->hidden + 255) / 256;
  ProfScope ps(stream);
#define UB_LAUNCH(BF, NVV) embed_rows_fwd_kernel<BF, NVV><<<grid, 256, 0, stream>>>(p)
  if (a->dtype == UB200_BF16) {
    switch (nv) { case 1: UB_LAUNCH(true, 1); break; case 2: UB_LAUNCH(true, 2); break;
                  case 3: UB_LAUNCH(true, 3); break; default: UB_LAUNCH(true, 4); break; }
  } else {
    switch (nv) { case 1: UB_LAUNCH(false, 1); break; case 2: UB_LAUNCH(false, 2); break;
                  case 3: UB_LAUNCH(false, 3); break; default: UB_LAUNCH(false, 4); break; }
  }
#undef UB_LAUNCH
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int ub200_embed_bwd_scatter(const void* du, const int32_t* kind, const int32_t* word_id,
                                       const int32_t* pos_id, void* d_word, float* d_pos, int32_t T,
                                       int32_t hidden, int32_t dtype, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(du && kind && word_id && pos_id && d_word && d_pos, "embed_bwd_scatter: null pointer");
  UB_CHECK_ARG(T > 0 && hidden > 0 && hidden % 8 == 0, "embed_bwd_scatter: need T > 0, hidden %% 8 == 0");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (deterministic()) {
    UB_CHECK_ARG(hidden <= 1024, "embed_bwd_scatter: deterministic mode needs hidden <= 1024");
    ProfScope ps(stream);
    if (dtype == UB200_BF16)
      UB_CHECK_CUDA(launch_pdl(embed_bwd_scatter_det_kernel<true>, dim3(T, 2), dim3(128), 0, stream, 1, du, kind,
                               word_id, pos_id, d_word, d_pos, T, hidden));
    else
      UB_CHECK_CUDA(launch_pdl(embed_bwd_scatter_det_kernel<false>, dim3(T, 2), dim3(128), 0, stream, 1, du, kind,
                               word_id, pos_id, d_word, d_pos, T, hidden));
    return 0;
  }
  const int grid = (T + 7) / 8;
  ProfScope ps(stream);
  if (dtype == UB200_BF16)
    UB_CHECK_CUDA(launch_pdl(embed_bwd_scatter_kernel<true>, dim3(grid), dim3(256), 0, stream, 1, du, kind,
                             word_id, pos_id, d_word, d_pos, T, hidden));
  else
    UB_CHECK_CUDA(launch_pdl(embed_bwd_scatter_kernel<false>, dim3(grid), dim3(256), 0, stream, 1, du, kind,
                             word_id, pos_id, d_word, d_pos, T, hidden));
  return 0;
}

extern "C" int ub200_embed_bwd_colsums(const ub200_embed_colsum_args* a, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(a && a->x && a->out, "embed_bwd_colsums: null pointer");
  UB_CHECK_ARG(a->T > 0 && a->hidden > 0 && a->hidden % 8 == 0, "embed_bwd_colsums: need T > 0, hidden %% 8 == 0");
  UB_CHECK_ARG(a->mode == 0 || a->mode == 1, "embed_bwd_colsums: bad mode %d", a->mode);
  UB_CHECK_ARG(a->mode != 0 || (a->type_id && a->type_vocab > 0), "embed_bwd_colsums: mode 0 needs type_id / type_vocab");
  UB_CHECK_ARG(a->mode != 1 || (a->kind && a->img_src && a->pos_feat), "embed_bwd_colsums: mode 1 needs kind / img_src / pos_feat");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  WColsumParams p{};
  p.x = a->x; p.type_id = a->type_id; p.kind = a->kind; p.img_src = a->img_src; p.pos_feat = a->pos_feat;
  p.out = a->out; p.T = a->T; p.N = a->hidden; p.mode = a->mode;
  const int gx = (a->hidden + 255) / 256;
  int gy = 32;                                   // few row slabs: W x hidden atomics per slab
  if (gy > (a->T + 63) / 64) gy = (a->T + 63) / 64;
  if (gy < 1) gy = 1;
  p.rows_per_cta = (a->T + gy - 1) / gy;
  const int total = a->mode == 0 ? a->type_vocab : 7;
  for (int base = 0; base < total; base += 8) {
    p.base = base;
    p.nweights = total - base < 8 ? total - base : 8;
    if (a->mode == 0) { p.stride_k = a->hidden; p.stride_n = 1; p.out = a->out + static_cast<long long>(base) * a->hidden; }
    else { p.stride_k = 1; p.stride_n = 7; }
    ProfScope ps(stream);
    if (deterministic()) {
      if (a->dtype == UB200_BF16)
        UB_CHECK_CUDA(launch_pdl(wcolsum_det_kernel<true>, dim3(a->hidden / 8), dim3(256), 0, stream, 1, p));
      else
        UB_CHECK_CUDA(launch_pdl(wcolsum_det_kernel<false>, dim3(a->hidden / 8), dim3(256), 0, stream, 1, p));
      continue;
    }
    if (a->dtype == UB200_BF16)
      UB_CHECK_CUDA(launch_pdl(wcolsum_kernel<true>, dim3(gx, gy), dim3(256), 0, stream, 1, p));
    else
      UB_CHECK_CUDA(launch_pdl(wcolsum_kernel<false>, dim3(gx, gy), dim3(256), 0, stream, 1, p));
  }
  return 0;
}
