// Callers either side of the encoder stack (SURVEY.md §8f rows 1 and 2):
//
//   ce_fwd / ce_bwd   fused softmax cross-entropy over the tied MLM decoder's [n, V] scores
//                     (model/pretrain.py:122-127: F.cross_entropy(prediction_scores, labels,
//                     reduction='none')): per-row log-sum-exp + loss in fp32 from the 16-bit
//                     scores; backward writes (softmax - onehot) * dloss IN PLACE over the scores,
//                     zeroing the padding columns [V, ld) that keep the row pitch a multiple of 8.
//   dgelu_mul         dpre = dy * gelu_erf'(pre): BertPredictionHeadTransform backward
//                     (model/layer.py:188-203) between its LayerNorm backward and dense dgrad.
//   sumsq / adamw     multi-tensor gradient norm and AdamW step with the reference's exact update
//                     (optim/adamw.py:77-101: bias-corrected step size, decoupled decay applied
//                     AFTER the Adam update) on fp32 master weights, fused with gradient
//                     unscaling, global-norm clipping (train_vqa.py:223-226) and the 16-bit
//                     model-weight refresh that apex O2 does as separate passes.
//   region_score      referring-expression head (model/re.py:69-90): Linear(H, 1) over each
//                     sample's region rows, masked_fill, cross-entropy or ranking hinge, and the
//                     backward with fixed-order weight-gradient sums (no float atomics).
//   wra               word-region alignment of ITM pre-training (model/ot.py): per image-text pair
//                     the cosine cost between its text and region rows, 50 IPOT iterations in
//                     shared memory, the transport distance and its backward (T held constant).
#include "common.h"
#include "ptx.cuh"

namespace ub {

template <bool kBF16>
__device__ __forceinline__ void h_unpack8(const uint4& u, float* f) {
  float2 t;
  t = Elem<kBF16>::unpack(u.x); f[0] = t.x; f[1] = t.y;
  t = Elem<kBF16>::unpack(u.y); f[2] = t.x; f[3] = t.y;
  t = Elem<kBF16>::unpack(u.z); f[4] = t.x; f[5] = t.y;
  t = Elem<kBF16>::unpack(u.w); f[6] = t.x; f[7] = t.y;
}
template <bool kBF16>
__device__ __forceinline__ uint4 h_pack8(const float* f) {
  uint4 u;
  u.x = Elem<kBF16>::pack(f[0], f[1]); u.y = Elem<kBF16>::pack(f[2], f[3]);
  u.z = Elem<kBF16>::pack(f[4], f[5]); u.w = Elem<kBF16>::pack(f[6], f[7]);
  return u;
}

// CTA-wide reductions (256 threads), result broadcast to every thread
__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r = fmaxf(r, red[w]);
  return r;
}
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) r += red[w];
  return r;
}

// ------------------------------------------------------------------------------ cross-entropy fwd
// One CTA per row.  The row (V x 2 bytes, 58 KB for the BERT vocabulary) is read twice (max, then
// sum of exp) and stays in L1 / L2 between the passes.
template <bool kBF16>
__global__ void __launch_bounds__(256)
ce_fwd_kernel(const void* __restrict__ logits_, long long ld, const long long* __restrict__ targets,
              float* __restrict__ loss, float* __restrict__ lse_out, int V) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  __shared__ float red[8];
  const int row = blockIdx.x;
  const T16* x = reinterpret_cast<const T16*>(logits_) + static_cast<long long>(row) * ld;
  const uint4* xv = reinterpret_cast<const uint4*>(x);
  const int nvec = (V + 7) >> 3;
  float m = -INFINITY;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    float f[8];
    h_unpack8<kBF16>(__ldg(xv + v), f);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (v * 8 + e < V) m = fmaxf(m, f[e]);
  }
  m = block_max(m, red);
  float s = 0.f;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    float f[8];
    h_unpack8<kBF16>(__ldg(xv + v), f);
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (v * 8 + e < V) s += __expf(f[e] - m);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float lse = m + logf(s);
    lse_out[row] = lse;
    const long long t = targets[row];
    loss[row] = (t >= 0 && t < V) ? lse - Elem<kBF16>::to_f(x[t]) : 0.f;
  }
}

// ------------------------------------------------------------------------------ cross-entropy bwd
// d[r, c] = (exp(x[r, c] - lse[r]) - [c == target[r]]) * dloss[r]; columns [V, ncols) -> 0.
// `out` may alias `logits` (each 16-byte vector is read and written by the same thread).
template <bool kBF16>
__global__ void __launch_bounds__(256)
ce_bwd_kernel(const void* logits_, void* out_, long long ld, const long long* __restrict__ targets,
              const float* __restrict__ lse, const float* __restrict__ dloss, int V, int ncols) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  const int row = blockIdx.x;
  const uint4* xv = reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(logits_) +
                                                   static_cast<long long>(row) * ld);
  uint4* ov = reinterpret_cast<uint4*>(reinterpret_cast<T16*>(out_) + static_cast<long long>(row) * ld);
  const long long t = targets[row];
  const bool live = t >= 0 && t < V;
  const float g = live ? dloss[row] : 0.f;
  const float l = lse[row];
  const int nvec = ncols >> 3;
  for (int v = threadIdx.x; v < nvec; v += 256) {
    float f[8];
    h_unpack8<kBF16>(xv[v], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = v * 8 + e;
      float d = 0.f;
      if (live && c < V) d = (__expf(f[e] - l) - (c == t ? 1.f : 0.f)) * g;
      f[e] = d;
    }
    ov[v] = h_pack8<kBF16>(f);
  }
}

// ------------------------------------------------------------------------------ dy * gelu'(pre)
// kTanh: out = dy * (1 - y^2) with y = tanh(pre) saved by the forward (BertPooler backward)
template <bool kBF16, bool kTanh = false>
__global__ void __launch_bounds__(256)
dgelu_mul_kernel(const uint4* __restrict__ dy, const uint4* __restrict__ pre, uint4* __restrict__ out,
                 long long nvec) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float a[8], b[8];
    h_unpack8<kBF16>(__ldg(dy + i), a);
    h_unpack8<kBF16>(__ldg(pre + i), b);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] *= kTanh ? (1.0f - b[e] * b[e]) : dgelu_erf(b[e]);
    out[i] = h_pack8<kBF16>(a);
  }
}

// ------------------------------------------------------------------------------ multi-tensor optimizer
// A segment is one parameter tensor.  CTA `b` owns elements [ (b - blk_start[s]) * ADAM_CHUNK, +ADAM_CHUNK )
// of the segment s with blk_start[s] <= b < blk_start[s + 1] (binary search over <= a few hundred
// segments).
constexpr int ADAM_CHUNK = 4096;   // elements per CTA: 256 threads x 16

__device__ __forceinline__ int find_segment(const int* __restrict__ blk_start, int nseg, int b) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(blk_start + mid) <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ float grad_of(const ub200_adam_segment& sg, long long i) {
  if (sg.grad_dtype == UB200_BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(sg.grad)[i]);
  if (sg.grad_dtype == UB200_F16) return __half2float(reinterpret_cast<const __half*>(sg.grad)[i]);
  return reinterpret_cast<const float*>(sg.grad)[i];
}

// sum of squares of all gradients (before unscaling) -> out[0] (fp32, atomically accumulated);
// kDet: each block's sum to out[blockIdx.x] instead
template <bool kDet>
__global__ void __launch_bounds__(256)
sumsq_kernel(const ub200_adam_segment* __restrict__ segs, const int* __restrict__ blk_start, int nseg,
             float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8];
  const int s = find_segment(blk_start, nseg, blockIdx.x);
  const ub200_adam_segment sg = segs[s];
  const long long base = static_cast<long long>(blockIdx.x - blk_start[s]) * ADAM_CHUNK;
  float acc = 0.f;
  if (sg.grad_dtype != UB200_F32 && sg.n % 8 == 0 && (reinterpret_cast<uintptr_t>(sg.grad) & 15) == 0) {
    const bool bf = sg.grad_dtype == UB200_BF16;
    for (int j = threadIdx.x * 8; j < ADAM_CHUNK; j += 2048) {
      const long long i = base + j;
      if (i >= sg.n) break;
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(sg.grad) + i));
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = bf ? Elem<true>::unpack(w[q]) : Elem<false>::unpack(w[q]);
        acc = fmaf(f.x, f.x, acc);
        acc = fmaf(f.y, f.y, acc);
      }
    }
  } else {
    for (int j = threadIdx.x; j < ADAM_CHUNK; j += 256) {
      const long long i = base + j;
      if (i < sg.n) { const float g = grad_of(sg, i); acc = fmaf(g, g, acc); }
    }
  }
  acc = block_sum(acc, red);
  if (kDet) {
    if (threadIdx.x == 0) out[blockIdx.x] = acc;   // partials[block]; summed by sumsq_finish_kernel
  } else if (threadIdx.x == 0 && acc != 0.f) {
    atomicAdd(out, acc);
  }
}

// Deterministic mode: out[0] += sum of partials[0 .. nblocks) in a fixed order (thread t sums blocks
// t, t + 256, ... ascending, then det_tree_sum8) -- the blocks are ADAM_CHUNK slices of the
// segments, so the result does not depend on the grid.
__global__ void __launch_bounds__(256)
sumsq_finish_kernel(const float* __restrict__ partials, int nblocks, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[256][9];
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < nblocks; b += 256) acc[0] += partials[b];
  const float s = det_tree_sum8(acc, red);
  if (threadIdx.x == 0) out[0] += s;
}

struct AdamHyper {
  float beta1, beta2, eps;
  float inv_scale;        // 1 / loss_scale (gradient unscaling)
  float max_norm;         // <= 0: no clipping
  const float* sumsq;     // device scalar from sumsq_kernel (of the SCALED gradients) or NULL
  const ub200_adam_state* state;   // device-resident step counter / overflow flag, or NULL (legacy)
  const float* lr;                 // per-group learning rates (device), with `state`
  const ub200_loss_scaler* scaler; // non-NULL: inv_scale is read from scaler->inv_scale instead
};

__device__ __forceinline__ bool sumsq_finite(float s) { return (s == s) && (fabsf(s) <= 3.0e38f); }

// found_inf / step bookkeeping on the device (one thread), between sumsq_kernel and adamw_kernel.
// No griddepcontrol, like adam_prep_scaled_kernel: an ordinary launch that never triggers early.
__global__ void adam_prep_kernel(const float* __restrict__ sumsq, ub200_adam_state* __restrict__ st) {
  const bool finite = sumsq_finite(*sumsq);
  st->found_inf = finite ? 0 : 1;
  if (finite) st->step += 1; else st->skipped += 1;
}

// adam_prep_kernel + apex's dynamic LossScaler.update_scale for the scaler entry of this step's loss:
// records the unscale factor of the gradients (1 / the scale their loss was multiplied by), then
// halves the scale on overflow (down to the optional floor) or doubles it after `window` clean steps
// (up to max_scale).  Only `sc` moves: the entries of the other losses are not touched.
// No griddepcontrol here (see ub200_adam_prep_scaled): launched behind sumsq_kernel with a full
// dependency, and never triggering early, so adamw_kernel can only start once it has finished.
__global__ void adam_prep_scaled_kernel(const float* __restrict__ sumsq, ub200_adam_state* __restrict__ st,
                                        ub200_loss_scaler* __restrict__ sc) {
  const bool finite = sumsq_finite(*sumsq);
  st->found_inf = finite ? 0 : 1;
  if (finite) st->step += 1; else st->skipped += 1;
  const float scale = sc->scale;
  sc->inv_scale = 1.0f / scale;
  if (!finite) {
    const float halved = scale * 0.5f;
    sc->scale = sc->min_scale > 0.f ? fmaxf(halved, sc->min_scale) : halved;
    sc->unskipped = 0;
  } else {
    int32_t u = sc->unskipped + 1;
    if (u == sc->window) {
      sc->scale = fminf(scale * 2.0f, sc->max_scale);
      u = 0;
    }
    sc->unskipped = u;
  }
}

__global__ void __launch_bounds__(256)
adamw_kernel(const ub200_adam_segment* __restrict__ segs, const int* __restrict__ blk_start, int nseg,
             const AdamHyper h) {
  pdl_launch_dependents();
  pdl_wait();
  const int s = find_segment(blk_start, nseg, blockIdx.x);
  const ub200_adam_segment sg = segs[s];
  const long long base = static_cast<long long>(blockIdx.x - blk_start[s]) * ADAM_CHUNK;
  float step_size = sg.step_size, lr_wd = sg.lr_wd;
  if (h.state != nullptr) {
    // an overflowed gradient (fp16 loss scaling) must not touch masters / moments / weights:
    // g * 0 would be NaN for g = inf (apex's dynamic scaler skips such a step)
    if (h.state->found_inf) return;
    const float lr = __ldg(h.lr + sg.group);
    step_size = lr;
    if (sg.flags & 1) {
      // once per CTA, in double: 1 - beta^t loses all its digits in fp32 for beta = 0.999, t = 1
      const double t = static_cast<double>(h.state->step - sg.step_offset);
      step_size = static_cast<float>(static_cast<double>(lr) * sqrt(1.0 - pow(static_cast<double>(h.beta2), t)) /
                                     (1.0 - pow(static_cast<double>(h.beta1), t)));
    }
    lr_wd = lr * sg.weight_decay;
  }
  const float inv_scale = h.scaler != nullptr ? h.scaler->inv_scale : h.inv_scale;
  float gmul = inv_scale;
  if (h.max_norm > 0.f && h.sumsq != nullptr) {
    // torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), applied iff < 1
    const float total = sqrtf(__ldg(h.sumsq)) * inv_scale;
    const float coef = h.max_norm / (total + 1e-6f);
    if (coef < 1.f) gmul *= coef;
  }
  auto update = [&](float g, float& m, float& v, float& p) {
    g *= gmul;
    m = m * h.beta1 + (1.0f - h.beta1) * g;              // optim/adamw.py:77
    v = v * h.beta2 + (1.0f - h.beta2) * g * g;          // :78
    const float denom = sqrtf(v) + h.eps;                // :79
    p = p - step_size * (m / denom);                     // :81-88 (bias-corrected step size)
    if (lr_wd > 0.f) p = p - lr_wd * p;                  // :99-100 decoupled decay AFTER the update
  };
  // vector path: 4 elements per thread (16-byte fp32 accesses, 8-byte 16-bit accesses) when the
  // segment is a 16-bit parameter with a 16-bit gradient of the same type and everything is aligned
  const bool vec = (sg.n % 4 == 0) && sg.model != nullptr && sg.grad_dtype == sg.model_dtype &&
                   sg.grad_dtype != UB200_F32 &&
                   ((reinterpret_cast<uintptr_t>(sg.master) | reinterpret_cast<uintptr_t>(sg.exp_avg) |
                     reinterpret_cast<uintptr_t>(sg.exp_avg_sq)) & 15) == 0 &&
                   ((reinterpret_cast<uintptr_t>(sg.grad) | reinterpret_cast<uintptr_t>(sg.model)) & 7) == 0;
  if (vec) {
    const bool bf = sg.grad_dtype == UB200_BF16;
    for (int j = threadIdx.x * 4; j < ADAM_CHUNK; j += 1024) {
      const long long i = base + j;
      if (i >= sg.n) break;
      const uint2 graw = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(sg.grad) + i);
      float4 m4 = *reinterpret_cast<const float4*>(sg.exp_avg + i);
      float4 v4 = *reinterpret_cast<const float4*>(sg.exp_avg_sq + i);
      float4 p4 = *reinterpret_cast<const float4*>(sg.master + i);
      const float2 g01 = bf ? Elem<true>::unpack(graw.x) : Elem<false>::unpack(graw.x);
      const float2 g23 = bf ? Elem<true>::unpack(graw.y) : Elem<false>::unpack(graw.y);
      update(g01.x, m4.x, v4.x, p4.x);
      update(g01.y, m4.y, v4.y, p4.y);
      update(g23.x, m4.z, v4.z, p4.z);
      update(g23.y, m4.w, v4.w, p4.w);
      *reinterpret_cast<float4*>(sg.exp_avg + i) = m4;
      *reinterpret_cast<float4*>(sg.exp_avg_sq + i) = v4;
      *reinterpret_cast<float4*>(sg.master + i) = p4;
      uint2 o;
      o.x = bf ? Elem<true>::pack(p4.x, p4.y) : Elem<false>::pack(p4.x, p4.y);
      o.y = bf ? Elem<true>::pack(p4.z, p4.w) : Elem<false>::pack(p4.z, p4.w);
      *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(sg.model) + i) = o;
    }
    return;
  }
  for (int j = threadIdx.x; j < ADAM_CHUNK; j += 256) {
    const long long i = base + j;
    if (i >= sg.n) break;
    float m = sg.exp_avg[i], v = sg.exp_avg_sq[i], p = sg.master[i];
    update(grad_of(sg, i), m, v, p);
    sg.exp_avg[i] = m; sg.exp_avg_sq[i] = v; sg.master[i] = p;
    if (sg.model) {
      if (sg.model_dtype == UB200_BF16) reinterpret_cast<__nv_bfloat16*>(sg.model)[i] = __float2bfloat16_rn(p);
      else if (sg.model_dtype == UB200_F16) reinterpret_cast<__half*>(sg.model)[i] = __float2half_rn(p);
      else reinterpret_cast<float*>(sg.model)[i] = p;
    }
  }
}

// ------------------------------------------------------------------------------ referring expressions
// model/re.py:69-90: re_output (Linear(H, 1)) over each sample's region rows, masked_fill(obj_masks,
// -1e4), then CrossEntropyLoss or the sigmoid ranking hinge.  One CTA per sample (<= ~100 regions).
constexpr int RE_THREADS = 256;
constexpr int RE_MAX_REGIONS = 8192;   // scores of one sample in shared memory (32 KB)

__device__ __forceinline__ float re_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ bool re_live(const uint8_t* __restrict__ obj_masks, int b, int k, int len, int Smax) {
  return k < len && obj_masks[static_cast<long long>(b) * Smax + k] == 0;
}

// The ranking hinge margin + sigmoid(s_n) - sigmoid(s_t), recomputed bit for bit by the backward.
__device__ __forceinline__ float re_hinge(float margin, float s_neg, float s_pos) {
  return margin + re_sigmoid(s_neg) - re_sigmoid(s_pos);
}

template <bool kBF16>
__global__ void __launch_bounds__(RE_THREADS)
region_score_fwd_kernel(const ub200_region_score_args a) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  extern __shared__ float re_sc[];          // [Smax] rounded scores
  __shared__ float red[8];
  const int b = blockIdx.x, Smax = a.max_regions, H = a.hidden;
  const int start = a.seg_start[b], len = a.seg_len[b];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint4* wv = reinterpret_cast<const uint4*>(a.weight);
  const float bias = a.bias != nullptr ? Elem<kBF16>::to_f(*reinterpret_cast<const T16*>(a.bias)) : 0.f;
  const float masked = Elem<kBF16>::to_f(Elem<kBF16>::from_f(-1e4f));
  // one warp per region: lane-strided 16-byte vectors, fp32 FMA chains, then a fixed xor tree
  for (int k = warp; k < Smax; k += RE_THREADS / 32) {
    float s = masked;
    if (re_live(a.obj_masks, b, k, len, Smax)) {
      const uint4* hv = reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(a.rows) +
                                                       static_cast<long long>(start + k) * H);
      float acc = 0.f;
      for (int v = lane; v < (H >> 3); v += 32) {
        float h[8], w[8];
        h_unpack8<kBF16>(__ldg(hv + v), h);
        h_unpack8<kBF16>(__ldg(wv + v), w);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc = fmaf(h[e], w[e], acc);
      }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      s = Elem<kBF16>::to_f(Elem<kBF16>::from_f(acc + bias));
    }
    if (lane == 0) re_sc[k] = s;
  }
  __syncthreads();
  T16* out = reinterpret_cast<T16*>(a.scores) + static_cast<long long>(b) * Smax;
  for (int k = threadIdx.x; k < Smax; k += RE_THREADS) out[k] = Elem<kBF16>::from_f(re_sc[k]);
  if (a.mode == UB200_RE_SCORES) return;
  const long long t = a.targets[b];
  const bool tvalid = t >= 0 && t < len;
  if (a.mode == UB200_RE_CLS) {
    // CrossEntropyLoss over the whole masked row: masked positions hold -1e4 and add exp(-1e4 - m) = 0
    float m = -INFINITY;
    for (int k = threadIdx.x; k < Smax; k += RE_THREADS) m = fmaxf(m, re_sc[k]);
    m = block_max(m, red);
    float s = 0.f;
    for (int k = threadIdx.x; k < Smax; k += RE_THREADS) s += expf(re_sc[k] - m);
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
      const float lse = m + logf(s);
      a.lse[b] = lse;
      a.loss[b] = tvalid ? lse - re_sc[t] : 0.f;
    }
    return;
  }
  if (threadIdx.x != 0) return;
  int n = -1;
  if (tvalid) {
    const long long p = a.neg_plan[b];
    if (p >= 0) {
      if (p < len && p != t) n = static_cast<int>(p);
    } else {
      // hard negative (model/re.py:115-121): the best region != t, unmasked ones first, ties to the
      // lowest index; a sample whose other regions are all masked falls back to its lowest other index
      bool best_live = false;
      float best = 0.f;
      for (int k = 0; k < len; ++k) {
        if (k == t) continue;
        const bool live = re_live(a.obj_masks, b, k, len, Smax);
        if (n < 0 || (live && !best_live) || (live == best_live && re_sc[k] > best)) {
          n = k;
          best = re_sc[k];
          best_live = live;
        }
      }
    }
  }
  a.neg_ix[b] = n;
  a.loss[b] = n >= 0 ? fmaxf(re_hinge(a.margin, re_sc[n], re_sc[t]), 0.f) : 0.f;
}

// dscore into shared memory, then per column vector: d_rows = dscore * w over the segment's rows and
// the sample's partial of dweight (rows in ascending order); padding rows after the segment (and
// before the first one) are zeroed by the CTA that owns the preceding segment.
template <bool kBF16>
__global__ void __launch_bounds__(RE_THREADS)
region_score_bwd_kernel(const ub200_region_score_args a) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  extern __shared__ float re_ds[];          // [Smax] dscore
  const int b = blockIdx.x, Smax = a.max_regions, H = a.hidden;
  const int start = a.seg_start[b], len = a.seg_len[b];
  const T16* sc = reinterpret_cast<const T16*>(a.scores) + static_cast<long long>(b) * Smax;
  const long long t = a.targets[b];
  const bool tvalid = t >= 0 && t < len;
  const float g = a.dloss[b];
  float* part_w = reinterpret_cast<float*>(a.workspace);
  float* part_b = part_w + static_cast<long long>(a.batch) * H;
  const float lse = a.mode == UB200_RE_CLS ? a.lse[b] : 0.f;
  for (int k = threadIdx.x; k < Smax; k += RE_THREADS) {
    float d = 0.f;
    if (a.mode == UB200_RE_CLS && tvalid && re_live(a.obj_masks, b, k, len, Smax))
      d = (expf(Elem<kBF16>::to_f(sc[k]) - lse) - (k == t ? 1.f : 0.f)) * g;
    re_ds[k] = d;
  }
  __syncthreads();
  if (a.mode == UB200_RE_RANK && threadIdx.x == 0) {
    const int n = a.neg_ix[b];
    if (tvalid && n >= 0) {
      const float sn = Elem<kBF16>::to_f(sc[n]), sp = Elem<kBF16>::to_f(sc[t]);
      if (re_hinge(a.margin, sn, sp) >= 0.f) {     // torch.clamp passes the gradient at 0
        const float gn = re_sigmoid(sn), gp = re_sigmoid(sp);
        if (re_live(a.obj_masks, b, n, len, Smax)) re_ds[n] = gn * (1.f - gn) * g;
        if (re_live(a.obj_masks, b, static_cast<int>(t), len, Smax)) re_ds[t] = -gp * (1.f - gp) * g;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < Smax; ++k) s += re_ds[k];
    part_b[b] = s;
  }
  const uint4* wv = reinterpret_cast<const uint4*>(a.weight);
  const T16* rows = reinterpret_cast<const T16*>(a.rows);
  T16* drows = reinterpret_cast<T16*>(a.d_rows);
  const int nvec = H >> 3;
  for (int v = threadIdx.x; v < nvec; v += RE_THREADS) {
    float w[8], acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    h_unpack8<kBF16>(__ldg(wv + v), w);
    for (int k = 0; k < len; ++k) {
      const long long r = static_cast<long long>(start + k) * H;
      const float d = re_ds[k];
      float h[8], o[8];
      h_unpack8<kBF16>(__ldg(reinterpret_cast<const uint4*>(rows + r) + v), h);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        acc[e] = fmaf(d, h[e], acc[e]);
        o[e] = d * w[e];
      }
      reinterpret_cast<uint4*>(drows + r)[v] = h_pack8<kBF16>(o);
    }
    float4* pw = reinterpret_cast<float4*>(part_w + static_cast<long long>(b) * H + v * 8);
    pw[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    pw[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
  const int gap_end = b + 1 < a.batch ? a.seg_start[b + 1] : a.R;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  auto zero_rows = [&](int lo, int hi) {
    for (long long i = static_cast<long long>(lo) * nvec + threadIdx.x; i < static_cast<long long>(hi) * nvec;
         i += RE_THREADS)
      reinterpret_cast<uint4*>(drows)[i] = zero;
  };
  zero_rows(start + len, gap_end);
  if (b == 0) zero_rows(0, start);
}

// dweight[c] = sum_b part_w[b, c], dbias = sum_b part_b[b]: one thread per column, samples in order.
__global__ void __launch_bounds__(RE_THREADS)
region_score_wsum_kernel(const float* __restrict__ part_w, int batch, int H, float* __restrict__ dw,
                         float* __restrict__ db) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * RE_THREADS + threadIdx.x;
  if (c > H) return;
  const float* src = c < H ? part_w + c : part_w + static_cast<long long>(batch) * H;
  const int stride = c < H ? H : 1;
  float s = 0.f;
  for (int b = 0; b < batch; ++b) s += src[static_cast<long long>(b) * stride];
  if (c < H) dw[c] = s; else if (db != nullptr) db[0] = s;
}

// ------------------------------------------------------------------------------ word-region alignment
// model/ot.py:optimal_transport_dist with its defaults (beta 0.5, 50 iterations, k = 1), restricted to the
// valid n x m block of each pair: the reference's padded entries of A and T are zero, so its 1e4 padding
// terms never reach a valid entry.  Matrices are [n, m] (region-major, like the reference's T), entry
// e = j * m + i.
constexpr int WRA_THREADS = 256;
constexpr int WRA_ITERS = 50;
constexpr float WRA_BETA = 0.5f;
constexpr float WRA_EPS = 1e-5f;   // F.normalize eps of cost_matrix_cosine
constexpr int WRA_MAXV = 4;        // 16-byte vectors per lane of a row: hidden <= 32 * 8 * 4

// workspace of pair b: T [max_m * max_n] then the raw row norms [max_m + max_n] (text, then regions)
__device__ __forceinline__ float* wra_pair_ws(const ub200_wra_args& a, int b) {
  const long long stride = static_cast<long long>(a.max_m) * a.max_n + a.max_m + a.max_n;
  return reinterpret_cast<float*>(a.workspace) + b * stride;
}

__device__ __forceinline__ bool wra_pair_ok(const ub200_wra_args& a, int m, int n) {
  return m >= 1 && n >= 1 && m <= a.max_m && n <= a.max_n;
}

// D += A (16x16, row) . B (16x8, col), 16-bit inputs, fp32 accumulation
template <bool kBF16>
__device__ __forceinline__ void mma_16816(float* d, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                          uint32_t b0, uint32_t b1) {
  if constexpr (kBF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Shared memory: C, A, P [max_m * max_n] (P holds Q, then T), sigma [max_m], delta [max_n], norms
// [max_m + max_n], column partials [256] (S * m <= 256 where S > 1).
template <bool kBF16>
__global__ void __launch_bounds__(WRA_THREADS)
wra_fwd_kernel(const ub200_wra_args a) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  extern __shared__ float wra_sm[];
  __shared__ float red[8];
  const int b = blockIdx.x, H = a.hidden, MN = a.max_m * a.max_n;
  const int start = a.cu_seqlens[b], m = a.txt_len[b], n = a.cu_seqlens[b + 1] - start - m;
  if (!wra_pair_ok(a, m, n)) {
    if (threadIdx.x == 0) a.dist[b] = __int_as_float(0x7fc00000);
    return;
  }
  float* C = wra_sm;
  float* A = C + MN;
  float* P = A + MN;
  float* sig = P + MN;
  float* del = sig + a.max_m;
  float* nrm = del + a.max_n;
  float* part = nrm + a.max_m + a.max_n;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, mn = m * n;
  const T16* X = reinterpret_cast<const T16*>(a.packed) + static_cast<long long>(start) * H;
  const T16* Y = X + static_cast<long long>(m) * H;

  // raw row norms in fp32: one warp per row, lane-strided 16-byte vectors, a fixed xor tree
  for (int r = warp; r < m + n; r += WRA_THREADS / 32) {
    const uint4* v = reinterpret_cast<const uint4*>(X + static_cast<long long>(r) * H);
    float s = 0.f;
    for (int c = lane; c < (H >> 3); c += 32) {
      float f[8];
      h_unpack8<kBF16>(__ldg(v + c), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) s = fmaf(f[e], f[e], s);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) nrm[r] = sqrtf(s);
  }
  // x_i . y_j: one warp per 16 x 8 tile, fragments loaded straight from global memory; rows past m / n
  // are clamped to the last valid row and their results dropped
  {
    const int g = lane >> 2, t4 = lane & 3, mb = (m + 15) >> 4, nb = (n + 7) >> 3;
    for (int tile = warp; tile < mb * nb; tile += WRA_THREADS / 32) {
      const int i0 = (tile / nb) * 16, j0 = (tile % nb) * 8;
      const uint32_t* xa = reinterpret_cast<const uint32_t*>(X + static_cast<long long>(min(i0 + g, m - 1)) * H) + t4;
      const uint32_t* xb = reinterpret_cast<const uint32_t*>(X + static_cast<long long>(min(i0 + g + 8, m - 1)) * H) + t4;
      const uint32_t* yb = reinterpret_cast<const uint32_t*>(Y + static_cast<long long>(min(j0 + g, n - 1)) * H) + t4;
      float d[4] = {0.f, 0.f, 0.f, 0.f};
      for (int k = 0; k < (H >> 1); k += 8)
        mma_16816<kBF16>(d, __ldg(xa + k), __ldg(xb + k), __ldg(xa + k + 4), __ldg(xb + k + 4), __ldg(yb + k),
                         __ldg(yb + k + 4));
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = i0 + g + (q >> 1) * 8, j = j0 + 2 * t4 + (q & 1);
        if (i < m && j < n) C[j * m + i] = d[q];
      }
    }
  }
  __syncthreads();
  for (int e = tid; e < mn; e += WRA_THREADS) {
    const int j = e / m, i = e - j * m;
    const float c = 1.f - C[e] * __frcp_rn(fmaxf(nrm[i], WRA_EPS) * fmaxf(nrm[m + j], WRA_EPS));
    C[e] = c;
    A[e] = expf(-c / WRA_BETA);
  }
  for (int i = tid; i < m; i += WRA_THREADS) sig[i] = __frcp_rn(static_cast<float>(m));
  __syncthreads();

  // IPOT.  T = delta * Q * sigma of one iteration is folded into the next one's Q = A * T (the same
  // products in the same order as the two steps).  sigma's column sums run over `S` slices of the
  // regions, added in slice order.
  const float fm = static_cast<float>(m), fn = static_cast<float>(n);
  const int S = m < WRA_THREADS ? WRA_THREADS / m : 1, jper = (n + S - 1) / S;
  for (int it = 0; it < WRA_ITERS; ++it) {
    for (int j = warp; j < n; j += WRA_THREADS / 32) {
      float s = 0.f;
      for (int i = lane; i < m; i += 32) {
        const int e = j * m + i;
        const float q = it == 0 ? A[e] : A[e] * (del[j] * P[e] * sig[i]);
        P[e] = q;
        s = fmaf(q, sig[i], s);
      }
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      __syncwarp();
      if (lane == 0) del[j] = __frcp_rn(fn * s);
    }
    __syncthreads();
    for (int c = tid; c < S * m; c += WRA_THREADS) {
      const int sl = c / m, i = c - sl * m;
      float s = 0.f;
      for (int j = sl * jper; j < min(n, (sl + 1) * jper); ++j) s = fmaf(del[j], P[j * m + i], s);
      if (S == 1) sig[i] = __frcp_rn(fm * s);
      else part[c] = s;
    }
    __syncthreads();
    if (S > 1) {
      for (int i = tid; i < m; i += WRA_THREADS) {
        float s = part[i];
        for (int sl = 1; sl < S; ++sl) s += part[sl * m + i];
        sig[i] = __frcp_rn(fm * s);
      }
      __syncthreads();
    }
  }
  float* ws = wra_pair_ws(a, b);
  float dist = 0.f;
  for (int e = tid; e < mn; e += WRA_THREADS) {
    const int j = e / m, i = e - j * m;
    const float t = del[j] * P[e] * sig[i];
    ws[e] = t;
    dist = fmaf(C[e], t, dist);
  }
  for (int r = tid; r < m + n; r += WRA_THREADS) ws[MN + r] = nrm[r];
  dist = block_sum(dist, red);
  if (tid == 0) a.dist[b] = Elem<kBF16>::to_f(Elem<kBF16>::from_f(dist));
}

// One output row pair per warp iteration: d(own row) = normalize-backward(-g sum_k w_k other_k), with
// w_k = T[k, i] / |y_k| for a text row i (other = regions) and T[j, k] / |x_k| for a region row j.
template <bool kBF16>
__device__ __forceinline__ void wra_bwd_rows(const ub200_wra_args& a, const float* P, const float* nrm, int m,
                                             int n, const typename Elem<kBF16>::T* X, bool text, int o0,
                                             float g, typename Elem<kBF16>::T* dX) {
  using T16 = typename Elem<kBF16>::T;
  const int H = a.hidden, lane = threadIdx.x & 31, nvec = H >> 3;
  const int own_n = text ? m : n, K = text ? n : m;
  const T16* own = text ? X : X + static_cast<long long>(m) * H;
  const T16* other = text ? X + static_cast<long long>(m) * H : X;
  const float* onrm = text ? nrm + m : nrm;
  const bool two = o0 + 1 < own_n;
  float acc[2][WRA_MAXV][8];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int v = 0; v < WRA_MAXV; ++v)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[r][v][e] = 0.f;
  for (int k = 0; k < K; ++k) {
    const float inv = __frcp_rn(fmaxf(onrm[k], WRA_EPS));
    const float w0 = (text ? P[k * m + o0] : P[o0 * m + k]) * inv;
    const float w1 = two ? (text ? P[k * m + o0 + 1] : P[(o0 + 1) * m + k]) * inv : 0.f;
    const uint4* ov = reinterpret_cast<const uint4*>(other + static_cast<long long>(k) * H);
#pragma unroll
    for (int v = 0; v < WRA_MAXV; ++v) {
      if (lane + 32 * v < nvec) {
        float f[8];
        h_unpack8<kBF16>(__ldg(ov + lane + 32 * v), f);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          acc[0][v][e] = fmaf(w0, f[e], acc[0][v][e]);
          acc[1][v][e] = fmaf(w1, f[e], acc[1][v][e]);
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (r == 1 && !two) break;
    const int o = o0 + r;
    const float nr = (text ? nrm : nrm + m)[o], s = fmaxf(nr, WRA_EPS), inv = __frcp_rn(s);
    const uint4* xv = reinterpret_cast<const uint4*>(own + static_cast<long long>(o) * H);
    float xs[WRA_MAXV][8];
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < WRA_MAXV; ++v) {
      if (lane + 32 * v < nvec) {
        h_unpack8<kBF16>(__ldg(xv + lane + 32 * v), xs[v]);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          acc[r][v][e] *= -g;                          // d(x^) = -g sum_k w_k other_k
          dot = fmaf(acc[r][v][e], xs[v][e], dot);
        }
      }
    }
#pragma unroll
    for (int q = 16; q >= 1; q >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, q);
    // x / max(|x|, eps): the norm's gradient flows only where |x| >= eps (clamp_min)
    const float coef = nr >= WRA_EPS ? dot / (s * s * s) : 0.f;
    uint4* dv = reinterpret_cast<uint4*>((text ? dX : dX + static_cast<long long>(m) * H) +
                                         static_cast<long long>(o) * H);
#pragma unroll
    for (int v = 0; v < WRA_MAXV; ++v) {
      if (lane + 32 * v < nvec) {
        float out[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) out[e] = acc[r][v][e] * inv - coef * xs[v][e];
        dv[lane + 32 * v] = h_pack8<kBF16>(out);
      }
    }
  }
}

// Shared memory: T [max_m * max_n] and the norms [max_m + max_n] of the pair.  Rows from
// cu_seqlens[batch] on are zeroed by the last CTA.
template <bool kBF16>
__global__ void __launch_bounds__(WRA_THREADS)
wra_bwd_kernel(const ub200_wra_args a) {
  pdl_launch_dependents();
  pdl_wait();
  using T16 = typename Elem<kBF16>::T;
  extern __shared__ float wra_sm[];
  const int b = blockIdx.x, H = a.hidden, MN = a.max_m * a.max_n, nvec = H >> 3;
  const int start = a.cu_seqlens[b], end = a.cu_seqlens[b + 1], m = a.txt_len[b], n = end - start - m;
  const int tid = threadIdx.x, warp = tid >> 5;
  T16* dX = reinterpret_cast<T16*>(a.d_packed) + static_cast<long long>(start) * H;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  if (b == a.batch - 1)
    for (long long i = static_cast<long long>(end) * nvec + tid; i < static_cast<long long>(a.total_rows) * nvec;
         i += WRA_THREADS)
      reinterpret_cast<uint4*>(a.d_packed)[i] = zero;
  if (!wra_pair_ok(a, m, n)) {
    for (long long i = tid; i < static_cast<long long>(max(end - start, 0)) * nvec; i += WRA_THREADS)
      reinterpret_cast<uint4*>(dX)[i] = zero;
    return;
  }
  float* P = wra_sm;
  float* nrm = P + MN;
  const float* ws = wra_pair_ws(a, b);
  for (int e = tid; e < m * n; e += WRA_THREADS) P[e] = ws[e];
  for (int r = tid; r < m + n; r += WRA_THREADS) nrm[r] = ws[MN + r];
  __syncthreads();
  const float g = a.d_dist[b];
  const T16* X = reinterpret_cast<const T16*>(a.packed) + static_cast<long long>(start) * H;
  const int mu = (m + 1) >> 1, nu = (n + 1) >> 1;
  for (int u = warp; u < mu + nu; u += WRA_THREADS / 32) {
    if (u < mu) wra_bwd_rows<kBF16>(a, P, nrm, m, n, X, true, 2 * u, g, dX);
    else wra_bwd_rows<kBF16>(a, P, nrm, m, n, X, false, 2 * (u - mu), g, dX);
  }
}

}  // namespace ub

// ------------------------------------------------------------------------------ C ABI
extern "C" int ub200_ce_fwd(const void* logits, int64_t ld, const int64_t* targets, float* loss,
                            float* lse, int32_t rows, int32_t vocab, int32_t dtype,
                            ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(logits && targets && loss && lse, "ce_fwd: null pointer");
  UB_CHECK_ARG(rows > 0 && vocab > 0 && ld % 8 == 0 && ld >= (vocab + 7) / 8 * 8,
               "ce_fwd: need rows > 0, vocab > 0, ld %% 8 == 0 and ld >= vocab rounded up to 8");
  UB_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 15) == 0, "ce_fwd: logits must be 16-byte aligned");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(stream);
  const long long* tg = reinterpret_cast<const long long*>(targets);
  if (dtype == UB200_BF16)
    UB_CHECK_CUDA(launch_pdl(ce_fwd_kernel<true>, dim3(rows), dim3(256), 0, stream, 1, logits,
                             static_cast<long long>(ld), tg, loss, lse, vocab));
  else
    UB_CHECK_CUDA(launch_pdl(ce_fwd_kernel<false>, dim3(rows), dim3(256), 0, stream, 1, logits,
                             static_cast<long long>(ld), tg, loss, lse, vocab));
  return 0;
}

extern "C" int ub200_ce_bwd(const void* logits, void* dlogits, int64_t ld, const int64_t* targets,
                            const float* lse, const float* dloss, int32_t rows, int32_t vocab,
                            int32_t ncols, int32_t dtype, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(logits && dlogits && targets && lse && dloss, "ce_bwd: null pointer");
  UB_CHECK_ARG(rows > 0 && vocab > 0 && ncols % 8 == 0 && ncols >= vocab && ld % 8 == 0 && ld >= ncols,
               "ce_bwd: need vocab <= ncols <= ld, ncols %% 8 == 0, ld %% 8 == 0");
  UB_CHECK_ARG((reinterpret_cast<uintptr_t>(logits) & 15) == 0 && (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0,
               "ce_bwd: buffers must be 16-byte aligned");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(stream);
  const long long* tg = reinterpret_cast<const long long*>(targets);
  if (dtype == UB200_BF16)
    UB_CHECK_CUDA(launch_pdl(ce_bwd_kernel<true>, dim3(rows), dim3(256), 0, stream, 1, logits, dlogits,
                             static_cast<long long>(ld), tg, lse, dloss, vocab, ncols));
  else
    UB_CHECK_CUDA(launch_pdl(ce_bwd_kernel<false>, dim3(rows), dim3(256), 0, stream, 1, logits, dlogits,
                             static_cast<long long>(ld), tg, lse, dloss, vocab, ncols));
  return 0;
}

extern "C" int ub200_dgelu_mul(const void* dy, const void* pre, void* out, int64_t n, int32_t dtype,
                               ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(dy && pre && out, "dgelu_mul: null pointer");
  UB_CHECK_ARG(n > 0 && n % 8 == 0, "dgelu_mul: n must be a positive multiple of 8");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long nvec = n / 8;
  long long blocks = (nvec + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  ProfScope ps(stream);
  if (dtype == UB200_BF16)
    UB_CHECK_CUDA(launch_pdl(dgelu_mul_kernel<true>, dim3(static_cast<int>(blocks)), dim3(256), 0, stream, 1,
                             reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint4*>(pre),
                             reinterpret_cast<uint4*>(out), nvec));
  else
    UB_CHECK_CUDA(launch_pdl(dgelu_mul_kernel<false>, dim3(static_cast<int>(blocks)), dim3(256), 0, stream, 1,
                             reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint4*>(pre),
                             reinterpret_cast<uint4*>(out), nvec));
  return 0;
}

extern "C" int ub200_dtanh_mul(const void* dy, const void* y, void* out, int64_t n, int32_t dtype,
                               ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(dy && y && out, "dtanh_mul: null pointer");
  UB_CHECK_ARG(n > 0 && n % 8 == 0, "dtanh_mul: n must be a positive multiple of 8");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long long nvec = n / 8;
  long long blocks = (nvec + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  ProfScope ps(stream);
  if (dtype == UB200_BF16)
    UB_CHECK_CUDA(launch_pdl(dgelu_mul_kernel<true, true>, dim3(static_cast<int>(blocks)), dim3(256), 0, stream, 1,
                             reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint4*>(y),
                             reinterpret_cast<uint4*>(out), nvec));
  else
    UB_CHECK_CUDA(launch_pdl(dgelu_mul_kernel<false, true>, dim3(static_cast<int>(blocks)), dim3(256), 0, stream, 1,
                             reinterpret_cast<const uint4*>(dy), reinterpret_cast<const uint4*>(y),
                             reinterpret_cast<uint4*>(out), nvec));
  return 0;
}

extern "C" int32_t ub200_adam_chunk(void) { return ub::ADAM_CHUNK; }

extern "C" int ub200_grad_sumsq(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev,
                                int32_t nseg, int32_t nblocks, float* out, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(segs_dev && blk_start_dev && out && nseg > 0 && nblocks > 0, "grad_sumsq: bad argument");
  UB_CHECK_ARG(!deterministic(), "grad_sumsq: deterministic mode needs ub200_grad_sumsq_ws");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(stream);
  UB_CHECK_CUDA(launch_pdl(sumsq_kernel<false>, dim3(nblocks), dim3(256), 0, stream, 1, segs_dev, blk_start_dev,
                           nseg, out));
  return 0;
}

extern "C" int64_t ub200_grad_sumsq_workspace_bytes(int32_t nblocks) {
  return nblocks > 0 ? static_cast<int64_t>(nblocks) * 4 : 0;
}

extern "C" int ub200_grad_sumsq_ws(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev,
                                   int32_t nseg, int32_t nblocks, float* out, void* workspace,
                                   int64_t workspace_bytes, ub200_stream_t stream_) {
  using namespace ub;
  if (!deterministic()) return ub200_grad_sumsq(segs_dev, blk_start_dev, nseg, nblocks, out, stream_);
  UB_CHECK_ARG(segs_dev && blk_start_dev && out && nseg > 0 && nblocks > 0, "grad_sumsq: bad argument");
  UB_CHECK_ARG(workspace && (reinterpret_cast<uintptr_t>(workspace) & 3) == 0, "grad_sumsq: bad workspace");
  UB_CHECK_ARG(workspace_bytes >= ub200_grad_sumsq_workspace_bytes(nblocks),
               "grad_sumsq: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
               (long long)ub200_grad_sumsq_workspace_bytes(nblocks));
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  float* partials = reinterpret_cast<float*>(workspace);
  {
    ProfScope ps(stream);
    UB_CHECK_CUDA(launch_pdl(sumsq_kernel<true>, dim3(nblocks), dim3(256), 0, stream, 1, segs_dev, blk_start_dev,
                             nseg, partials));
  }
  ProfScope ps(stream);
  UB_CHECK_CUDA(launch_pdl(sumsq_finish_kernel, dim3(1), dim3(256), 0, stream, 1,
                           static_cast<const float*>(partials), nblocks, out));
  return 0;
}

extern "C" int ub200_adam_prep(const float* sumsq, ub200_adam_state* state_dev, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(sumsq && state_dev, "adam_prep: null pointer");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(stream);
  // An ordinary launch, for the reason given in ub200_adam_prep_scaled: chained by PDL inside a
  // captured graph, found_inf and the clip factor could read an incomplete sum of squares.
  adam_prep_kernel<<<1, 1, 0, stream>>>(sumsq, state_dev);
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int ub200_adamw_step(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev,
                                int32_t nseg, int32_t nblocks, float beta1, float beta2, float eps,
                                float inv_scale, float max_norm, const float* sumsq,
                                const ub200_adam_state* state_dev, const float* lr_dev,
                                ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(segs_dev && blk_start_dev && nseg > 0 && nblocks > 0, "adamw_step: bad argument");
  UB_CHECK_ARG((state_dev == nullptr) == (lr_dev == nullptr), "adamw_step: state_dev and lr_dev go together");
  UB_CHECK_ARG(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f,
               "adamw_step: invalid hyper-parameters");
  UB_CHECK_ARG(max_norm <= 0.f || sumsq, "adamw_step: clipping needs the sumsq scalar");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  AdamHyper h{beta1, beta2, eps, inv_scale, max_norm, sumsq, state_dev, lr_dev, nullptr};
  ProfScope ps(stream);
  UB_CHECK_CUDA(launch_pdl(adamw_kernel, dim3(nblocks), dim3(256), 0, stream, 1, segs_dev, blk_start_dev,
                           nseg, h));
  return 0;
}

extern "C" int ub200_adam_prep_scaled(const float* sumsq, ub200_adam_state* state_dev,
                                      ub200_loss_scaler* scalers_dev, int32_t loss_id, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(sumsq && state_dev && scalers_dev, "adam_prep_scaled: null pointer");
  UB_CHECK_ARG(loss_id >= 0, "adam_prep_scaled: loss_id must be >= 0");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ProfScope ps(stream);
  // An ordinary launch, not a programmatic dependent of sumsq_kernel: inside a captured CUDA graph the
  // PDL-chained form was measured reading the sum of squares before sumsq_kernel had added the
  // non-finite part of it (an overflowed step counted as clean), and adamw_kernel, when this kernel
  // triggered its dependents early, reading a stale found_inf.  Full dependencies on both sides cost
  // one launch latency each per step.
  adam_prep_scaled_kernel<<<1, 1, 0, stream>>>(sumsq, state_dev, scalers_dev + loss_id);
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int ub200_adamw_step_scaled(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev,
                                       int32_t nseg, int32_t nblocks, float beta1, float beta2, float eps,
                                       float max_norm, const float* sumsq, const ub200_adam_state* state_dev,
                                       const float* lr_dev, const ub200_loss_scaler* scalers_dev,
                                       int32_t loss_id, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(segs_dev && blk_start_dev && nseg > 0 && nblocks > 0, "adamw_step_scaled: bad argument");
  UB_CHECK_ARG(state_dev && lr_dev && scalers_dev && loss_id >= 0,
               "adamw_step_scaled: needs state_dev, lr_dev, scalers_dev and loss_id >= 0");
  UB_CHECK_ARG(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f,
               "adamw_step_scaled: invalid hyper-parameters");
  UB_CHECK_ARG(max_norm <= 0.f || sumsq, "adamw_step_scaled: clipping needs the sumsq scalar");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  AdamHyper h{beta1, beta2, eps, 1.0f, max_norm, sumsq, state_dev, lr_dev, scalers_dev + loss_id};
  ProfScope ps(stream);
  UB_CHECK_CUDA(launch_pdl(adamw_kernel, dim3(nblocks), dim3(256), 0, stream, 1, segs_dev, blk_start_dev,
                           nseg, h));
  return 0;
}

// ------------------------------------------------------------------------------ referring expressions
extern "C" int64_t ub200_region_score_workspace_bytes(int32_t batch, int32_t hidden) {
  return batch > 0 && hidden > 0 ? static_cast<int64_t>(batch) * (hidden + 1) * 4 : 0;
}

static int re_check(const ub200_region_score_args* a, const char* who) {
  using namespace ub;
  UB_CHECK_ARG(a && a->rows && a->weight && a->seg_start && a->seg_len && a->obj_masks && a->scores,
               "%s: null pointer", who);
  UB_CHECK_ARG(a->batch > 0 && a->R >= 0 && a->hidden > 0 && a->hidden % 8 == 0, "%s: need batch > 0, R >= 0 and "
               "hidden a positive multiple of 8", who);
  UB_CHECK_ARG(a->max_regions > 0 && a->max_regions <= RE_MAX_REGIONS, "%s: max_regions %d outside [1, %d]", who,
               a->max_regions, RE_MAX_REGIONS);
  UB_CHECK_ARG(a->mode == UB200_RE_SCORES || a->mode == UB200_RE_CLS || a->mode == UB200_RE_RANK,
               "%s: unknown mode %d", who, a->mode);
  UB_CHECK_ARG(a->dtype == UB200_F16 || a->dtype == UB200_BF16, "%s: dtype must be F16 or BF16", who);
  UB_CHECK_ARG(((reinterpret_cast<uintptr_t>(a->rows) | reinterpret_cast<uintptr_t>(a->weight)) & 15) == 0,
               "%s: rows and weight must be 16-byte aligned", who);
  UB_CHECK_ARG(a->mode == UB200_RE_SCORES || a->targets, "%s: the losses need targets", who);
  return 0;
}

extern "C" int ub200_region_score_fwd(const ub200_region_score_args* a, ub200_stream_t stream_) {
  using namespace ub;
  if (int rc = re_check(a, "region_score_fwd")) return rc;
  UB_CHECK_ARG(a->mode == UB200_RE_SCORES || a->loss, "region_score_fwd: the losses need loss");
  UB_CHECK_ARG(a->mode != UB200_RE_CLS || a->lse, "region_score_fwd: cls needs lse");
  UB_CHECK_ARG(a->mode != UB200_RE_RANK || (a->neg_plan && a->neg_ix), "region_score_fwd: rank needs neg_plan "
               "and neg_ix");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const size_t smem = static_cast<size_t>(a->max_regions) * sizeof(float);
  ProfScope ps(stream);
  if (a->dtype == UB200_BF16)
    UB_CHECK_CUDA(launch_pdl(region_score_fwd_kernel<true>, dim3(a->batch), dim3(RE_THREADS), smem, stream, 1, *a));
  else
    UB_CHECK_CUDA(launch_pdl(region_score_fwd_kernel<false>, dim3(a->batch), dim3(RE_THREADS), smem, stream, 1, *a));
  return 0;
}

extern "C" int ub200_region_score_bwd(const ub200_region_score_args* a, ub200_stream_t stream_) {
  using namespace ub;
  if (int rc = re_check(a, "region_score_bwd")) return rc;
  UB_CHECK_ARG(a->mode != UB200_RE_SCORES, "region_score_bwd: needs a loss mode");
  UB_CHECK_ARG(a->dloss && a->d_rows && a->dweight && a->workspace, "region_score_bwd: null pointer");
  UB_CHECK_ARG(a->mode != UB200_RE_CLS || a->lse, "region_score_bwd: cls needs lse");
  UB_CHECK_ARG(a->mode != UB200_RE_RANK || a->neg_ix, "region_score_bwd: rank needs neg_ix");
  UB_CHECK_ARG((reinterpret_cast<uintptr_t>(a->d_rows) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0,
               "region_score_bwd: d_rows and workspace must be 16-byte aligned");
  UB_CHECK_ARG(a->workspace_bytes >= ub200_region_score_workspace_bytes(a->batch, a->hidden),
               "region_score_bwd: workspace of %lld bytes, %lld needed", (long long)a->workspace_bytes,
               (long long)ub200_region_score_workspace_bytes(a->batch, a->hidden));
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const size_t smem = static_cast<size_t>(a->max_regions) * sizeof(float);
  {
    ProfScope ps(stream);
    if (a->dtype == UB200_BF16)
      UB_CHECK_CUDA(launch_pdl(region_score_bwd_kernel<true>, dim3(a->batch), dim3(RE_THREADS), smem, stream, 1, *a));
    else
      UB_CHECK_CUDA(launch_pdl(region_score_bwd_kernel<false>, dim3(a->batch), dim3(RE_THREADS), smem, stream, 1, *a));
  }
  ProfScope ps(stream);
  const int grid = (a->hidden + 1 + RE_THREADS - 1) / RE_THREADS;
  UB_CHECK_CUDA(launch_pdl(region_score_wsum_kernel, dim3(grid), dim3(RE_THREADS), 0, stream, 1,
                           static_cast<const float*>(a->workspace), a->batch, a->hidden, a->dweight, a->dbias));
  return 0;
}

// ------------------------------------------------------------------------------ word-region alignment
extern "C" int64_t ub200_wra_workspace_bytes(int32_t batch, int32_t max_m, int32_t max_n) {
  if (batch <= 0 || max_m <= 0 || max_n <= 0) return 0;
  return static_cast<int64_t>(batch) * (static_cast<int64_t>(max_m) * max_n + max_m + max_n) * 4;
}

static int wra_check(const ub200_wra_args* a, const char* who) {
  using namespace ub;
  UB_CHECK_ARG(a && a->packed && a->cu_seqlens && a->txt_len && a->workspace, "%s: null pointer", who);
  UB_CHECK_ARG(a->batch > 0 && a->total_rows >= 0 && a->max_m >= 1 && a->max_n >= 1,
               "%s: need batch > 0, total_rows >= 0, max_m >= 1 and max_n >= 1", who);
  UB_CHECK_ARG(a->dtype == UB200_F16 || a->dtype == UB200_BF16, "%s: dtype must be F16 or BF16", who);
  UB_CHECK_ARG((reinterpret_cast<uintptr_t>(a->packed) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->workspace) & 15) == 0,
               "%s: packed and workspace must be 16-byte aligned", who);
  UB_CHECK_ARG(a->workspace_bytes >= ub200_wra_workspace_bytes(a->batch, a->max_m, a->max_n),
               "%s: workspace of %lld bytes, %lld needed", who, (long long)a->workspace_bytes,
               (long long)ub200_wra_workspace_bytes(a->batch, a->max_m, a->max_n));
  if (a->hidden <= 0 || a->hidden % 16 != 0 || a->hidden > 32 * 8 * WRA_MAXV)
    return set_error(UB200_EUNSUPPORTED, "%s: hidden %d is not a multiple of 16 up to %d", who, a->hidden,
                     32 * 8 * WRA_MAXV);
  if (static_cast<long long>(a->max_m) * a->max_n > UB200_WRA_MAX_MN)
    return set_error(UB200_EUNSUPPORTED, "%s: max_m * max_n = %d * %d exceeds %d", who, a->max_m, a->max_n,
                     UB200_WRA_MAX_MN);
  return 0;
}

template <typename K>
static int wra_launch(K kern, unsigned long long& configured, size_t smem, const ub200_wra_args* a,
                      cudaStream_t stream) {
  using namespace ub;
  if (first_use_on_device(configured))
    UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(4 * (5 * UB200_WRA_MAX_MN + 2 + WRA_THREADS))));
  ProfScope ps(stream);
  UB_CHECK_CUDA(launch_pdl(kern, dim3(a->batch), dim3(WRA_THREADS), smem, stream, 1, *a));
  return 0;
}

extern "C" int ub200_wra_fwd(const ub200_wra_args* a, ub200_stream_t stream_) {
  using namespace ub;
  if (int rc = wra_check(a, "wra_fwd")) return rc;
  UB_CHECK_ARG(a->dist, "wra_fwd: null dist");
  static unsigned long long cfg[2];
  const size_t mn = static_cast<size_t>(a->max_m) * a->max_n;
  const size_t smem = 4 * (3 * mn + 2 * (static_cast<size_t>(a->max_m) + a->max_n) + WRA_THREADS);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (a->dtype == UB200_BF16) return wra_launch(wra_fwd_kernel<true>, cfg[1], smem, a, stream);
  return wra_launch(wra_fwd_kernel<false>, cfg[0], smem, a, stream);
}

extern "C" int ub200_wra_bwd(const ub200_wra_args* a, ub200_stream_t stream_) {
  using namespace ub;
  if (int rc = wra_check(a, "wra_bwd")) return rc;
  UB_CHECK_ARG(a->d_dist && a->d_packed, "wra_bwd: null pointer");
  UB_CHECK_ARG((reinterpret_cast<uintptr_t>(a->d_packed) & 15) == 0, "wra_bwd: d_packed must be 16-byte aligned");
  static unsigned long long cfg[2];
  const size_t smem = 4 * (static_cast<size_t>(a->max_m) * a->max_n + a->max_m + a->max_n);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (a->dtype == UB200_BF16) return wra_launch(wra_bwd_kernel<true>, cfg[1], smem, a, stream);
  return wra_launch(wra_bwd_kernel<false>, cfg[0], smem, a, stream);
}
