// Fused variable-length multi-head self-attention for sm_90a (head_dim = 64).
//
// Replaces model/layer.py:80-100 of the reference (transpose_for_scores, QK^T, /sqrt(d), +mask,
// softmax, dropout, PV, permute+contiguous: ~10 launches over the padded [B,h,L,L] rectangle)
// with ONE kernel over the packed [T, 3H] QKV matrix.  Q/K/V tiles are TMA'd straight out of the
// packed QKV buffer (column offsets 0 / H / 2H select q / k / v, +64*head selects the head).
//   * S = Q K^T and O = P V run on wgmma with fp32 accumulators in registers; P is taken from the
//     S registers (the fp32 accumulator fragment of S is the 16-bit A fragment of P once packed);
//   * mask-by-omission: only the S_b valid keys of the sequence take part (the reference's
//     additive -10000 underflows to exactly 0 probability, so this is exact — SURVEY.md §8a E4);
//   * softmax in registers (the 4 lanes that share a row reduce with shuffles), exp2 with
//     1/sqrt(d) folded in; probabilities are rounded to 16 bit BEFORE P.V, as the reference's
//     fp16 softmax output is;
//   * Philox dropout on P regenerated (not stored) by the backward kernel;
//   * ctx is written directly in [T, H] layout; the row-wise log-sum-exp is saved for backward.
//
// Backward (autograd mirror of the same lines) recomputes P from Q, K and the saved LSE:
//   dV = Pd^T dO,  dPd = dO V^T,  dS = P o (mask o dPd / keep - delta),  delta = rowsum(dO o O)
//   dQ = scale * dS K,  dK = scale * dS^T Q
// with all five contractions on wgmma from the same four TMA tiles (Q, K, V, dO) and the Pd / dS
// tiles the softmax threads write to shared memory; the transposed operands (P^T, dS^T, V as
// [keys x d], ...) are read MN-major through the wgmma transpose bits, nothing is transposed in
// memory.
//
// Two kernel families, picked by the host from max_seqlen:
//   * max_seqlen <= 128 (the pre-training batches: S ~ 40-72): persistent one-warpgroup CTAs, one
//     work item = one (head, sequence), all contractions m64n64 over 64-row blocks of that sequence
//     only, the next item's tiles TMA'd into a second stage while the current one computes;
//   * longer sequences: one CTA of two warpgroups per 128-row tile, looping over 128-key blocks.
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ub {

constexpr int ATT_D = 64;          // head dim (both UNITER configs)
constexpr int ATT_BM = 128;        // query rows per CTA (two warpgroups of 64)
constexpr int ATT_BN = 128;        // keys per KV block
constexpr int ATT_TILE = ATT_BM * ATT_D * 2;   // 16 KB: one 128x64 16-bit tile
constexpr int ATT_MAXSEQ = 512;    // dropout index pitch == max_position_embeddings
constexpr int ATT_THREADS = 256;

struct AttnParams {
  const int* cu_seqlens;   // [B+1]
  int B, H, nheads, T;
  void* ctx;               // [T, H] 16-bit
  float* lse;              // [nheads, T]
  float scale;             // 1/sqrt(d)
  uint32_t drop_thr16;
  float drop_inv_keep;
  uint32_t seed_lo, seed_hi, stream_lo, stream_hi;
  // backward only
  const void* dctx;        // [T, H]
  void* dqkv;              // [T, 3H]
  float* dbias;            // [3H] fp32 column sums of dqkv (QKV bias gradient), accumulated; or NULL
  const unsigned long long* rng_dev;   // optional device-side dropout stream offset (graph replay)
};

// Accumulator fragment of wgmma m64nN (per warp 16 rows): register 4*jj + 2*e + t holds row
// (lane / 4) + 8 * e, column 8 * jj + 2 * (lane % 4) + t.

// Column sums over the 16 rows of a warp of a 64-column fragment (rows with ok0 / ok1 false count
// as zero): lanes with equal lane % 4 hold the same columns; lanes 0-3 add the totals to dst.
__device__ __forceinline__ void frag_colsum64_atomic(const float (&d)[32], bool ok0, bool ok1, float* dst,
                                                     int lane) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      float x = (ok0 ? d[4 * jj + t] : 0.f) + (ok1 ? d[4 * jj + 2 + t] : 0.f);
      x += __shfl_xor_sync(0xffffffffu, x, 4);
      x += __shfl_xor_sync(0xffffffffu, x, 8);
      x += __shfl_xor_sync(0xffffffffu, x, 16);
      if (lane < 4) atomicAdd(dst + 8 * jj + 2 * lane + t, x);
    }
  }
}

// The same column sums added to dst[64] in shared memory that only this warp writes (plain adds:
// shared-memory float atomics are CAS loops on sm_90).
__device__ __forceinline__ void frag_colsum64_warp(const float (&d)[32], bool ok0, bool ok1, float* dst, int lane) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      float x = (ok0 ? d[4 * jj + t] : 0.f) + (ok1 ? d[4 * jj + 2 + t] : 0.f);
      x += __shfl_xor_sync(0xffffffffu, x, 4);
      x += __shfl_xor_sync(0xffffffffu, x, 8);
      x += __shfl_xor_sync(0xffffffffu, x, 16);
      if (lane < 4) dst[8 * jj + 2 * lane + t] += x;
    }
  }
}

// row e of this thread's fragment pair, 64 columns, times `mul`, as 16-bit into out_row
template <bool kBF16>
__device__ __forceinline__ void store_frag_row(void* out_row, const float (&d)[32], int e, int q4, float mul) {
  uint32_t* o = reinterpret_cast<uint32_t*>(out_row);
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
    o[(8 * jj + 2 * q4) >> 1] = Elem<kBF16>::pack(d[4 * jj + 2 * e] * mul, d[4 * jj + 2 * e + 1] * mul);
}

// element index used to key the attention-probability dropout mask
__device__ __forceinline__ uint64_t attn_drop_group(int bh, int q, int key8) {
  return ((static_cast<uint64_t>(bh) * ATT_MAXSEQ + q) * ATT_MAXSEQ + key8) >> 3;
}

// Dropout bits of 4 consecutive 8-key groups [4 jb, 4 jb + 4) of one query row, which the 4 lanes
// of a quad share: lane q4 runs Philox once, for group 4 jb + q4, and the quad exchanges words so that
// every lane ends up with word q4 of each group's block — the 16-bit lanes of its two keys 2 q4 and
// 2 q4 + 1 (rand16_of(block, 2 q4 + t)).  w[t] belongs to group 4 jb + t.  All 32 lanes must call it.
__device__ __forceinline__ void quad_drop_words(const DropoutRng& rng, int bh, int q, int key_base, int jb,
                                                int lane, uint32_t (&w)[4]) {
  const int q4 = lane & 3;
  const uint4 r = rng.draw8(attn_drop_group(bh, q, key_base + 8 * (4 * jb + q4)));
  uint32_t got[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    // round k: every lane sends word (q4 - k) & 3 and reads lane (q4 + k) & 3 of its quad, which
    // sent exactly word q4 of group 4 jb + ((q4 + k) & 3)
    const int sw = (q4 - k) & 3;
    const uint32_t v = sw == 0 ? r.x : (sw == 1 ? r.y : (sw == 2 ? r.z : r.w));
    got[k] = __shfl_sync(0xffffffffu, v, (lane & ~3) | ((q4 + k) & 3));
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int k = (t - q4) & 3;
    w[t] = k == 0 ? got[0] : (k == 1 ? got[1] : (k == 2 ? got[2] : got[3]));
  }
}

__device__ __forceinline__ uint32_t rand16_half(uint32_t w, int t) { return t ? (w >> 16) : (w & 0xFFFFu); }

// write two consecutive 16-bit values (one 32-bit word) of row `r`, columns [col, col+2), into a
// K-major SWIZZLE_128B operand made of 64-column slabs of 128 rows x 128 B.
__device__ __forceinline__ void st_swz128_u32(uint8_t* base, int r, int col, uint32_t v) {
  const int slab = col >> 6;
  const int chunk = (col & 63) >> 3;
  uint8_t* p = base + slab * ATT_TILE + r * 128 + ((chunk ^ (r & 7)) << 4) + (col & 7) * 2;
  *reinterpret_cast<uint32_t*>(p) = v;
}

// delta = rowsum(dO o O) and the saved log-sum-exp (times log2 e) of `row` of the sequence, read
// straight from global; each of the 4 lanes of a row takes 16 of its 64 columns.  All 32 lanes call it.
template <bool kBF16>
__device__ __forceinline__ void row_delta_lse(const AttnParams& p, int seq0, int head, int row, bool ok, int q4,
                                              float& delta, float& lse2) {
  using T16 = typename Elem<kBF16>::T;
  float d = 0.f;
  lse2 = 0.f;
  if (ok) {
    const size_t off = static_cast<size_t>(seq0 + row) * p.H + head * ATT_D + 16 * q4;
    const uint4* g_do = reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.dctx) + off);
    const uint4* g_o = reinterpret_cast<const uint4*>(reinterpret_cast<const T16*>(p.ctx) + off);
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const uint4 a = __ldg(g_do + v), o = __ldg(g_o + v);
      float2 x, y;
      x = Elem<kBF16>::unpack(a.x); y = Elem<kBF16>::unpack(o.x); d += x.x * y.x + x.y * y.y;
      x = Elem<kBF16>::unpack(a.y); y = Elem<kBF16>::unpack(o.y); d += x.x * y.x + x.y * y.y;
      x = Elem<kBF16>::unpack(a.z); y = Elem<kBF16>::unpack(o.z); d += x.x * y.x + x.y * y.y;
      x = Elem<kBF16>::unpack(a.w); y = Elem<kBF16>::unpack(o.w); d += x.x * y.x + x.y * y.y;
    }
    lse2 = p.lse[static_cast<size_t>(head) * p.T + seq0 + row] * 1.4426950408889634f;
  }
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  d += __shfl_xor_sync(0xffffffffu, d, 2);
  delta = d;
}

// =====================================================================================
// Short sequences (max_seqlen <= 128).  One CTA = one warpgroup, persistent; a work item is one
// (head, sequence) pair, split into nb = ceil(S / 64) <= 2 blocks of 64 rows.  Every contraction is
// m64n64 over the keys / queries of that sequence and head alone.  Thread 0 TMA-loads an item's
// 64-row tiles (Q, K, V and, backward, dO) into a stage of two 8 KB slots per tensor:
//   * single-block item: one slot, so the next single-block item is loaded into the other slot
//     while this one computes (full barrier per slot; the slot is empty once the warpgroup has
//     passed the named barrier that ends the item that last used it);
//   * two-block item: both slots (rows 0-63 / 64-127 contiguous, i.e. one 128-row operand), loaded
//     once the previous item is done.
// =====================================================================================
constexpr int SH_TILE = 64 * ATT_D * 2;   // 8 KB: one 64 x 64 16-bit tile (one TMA box)
constexpr int SH_THREADS = 128;
constexpr int SH_MAXSEQ = 128;

// the warpgroup's own barrier (a CTA is one warpgroup)
__device__ __forceinline__ void wg_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

__device__ __forceinline__ int seq_blocks(const int* cu, int b) { return min((cu[b + 1] - cu[b] + 63) >> 6, 2); }

// Static schedule from cu_seqlens, computed identically by every thread (no host read, no state
// to reset between launches or graph replays).  Items are ordered head-major, (h, b), and cost
// nb^2 (the 64 x 64 tiles of S).  CTA c takes the items whose cumulative cost starts in
// [c W / G, (c + 1) W / G): balanced in cost and contiguous, so most of a CTA's items share a head
// (the QKV bias gradient is flushed once per head change).  Empty sequences are skipped.
struct ShortSched {
  const int* cu;
  int B, nheads, h, b;
  long long start, hi;

  __device__ bool valid() const { return h < nheads && start < hi; }
  __device__ int blocks() const { return seq_blocks(cu, b); }

  __device__ void init(const int* cu_, int B_, int nheads_, int lane) {
    cu = cu_; B = B_; nheads = nheads_;
    h = nheads; start = hi = 0;
    int wb = 0;   // cost of one head
    for (int b0 = 0; b0 < B; b0 += 32) {
      int c = b0 + lane < B ? seq_blocks(cu, b0 + lane) : 0;
      c *= c;
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
      wb += c;
    }
    if (wb == 0) return;
    const long long W = static_cast<long long>(nheads) * wb;
    const long long lo = W * blockIdx.x / gridDim.x;
    hi = W * (blockIdx.x + 1) / gridDim.x;
    if (lo >= hi) return;
    const int hh = static_cast<int>(lo / wb);
    const long long r = lo - static_cast<long long>(hh) * wb;
    // first sequence of head hh whose cost prefix is >= r (warp-parallel scan over b)
    int pref = 0;
    for (int b0 = 0; b0 < B; b0 += 32) {
      int c = b0 + lane < B ? seq_blocks(cu, b0 + lane) : 0;
      c *= c;
      int incl = c;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      const int excl = pref + incl - c;
      const unsigned m = __ballot_sync(0xffffffffu, b0 + lane < B && excl >= r);
      if (m) {
        const int L = __ffs(m) - 1;
        h = hh;
        b = b0 + L;
        start = static_cast<long long>(hh) * wb + __shfl_sync(0xffffffffu, excl, L);
        skip_empty();
        return;
      }
      pref += __shfl_sync(0xffffffffu, incl, 31);
    }
    h = hh + 1;
    b = 0;
    start = static_cast<long long>(h) * wb;
    skip_empty();
  }
  __device__ void step() {
    const int nb = blocks();
    start += nb * nb;
    if (++b == B) { b = 0; ++h; }
  }
  __device__ void skip_empty() {
    while (valid() && cu[b + 1] == cu[b]) step();
  }
  __device__ void next() { step(); skip_empty(); }
};

// Forward rows [64 qb, 64 qb + 64) of one item, NB key blocks: S in registers, P from the S
// fragment, O = P V, then ctx and lse out.
template <bool kBF16, int NB>
__device__ __forceinline__ void attn_fwd_short_rows(const AttnParams& p, uint32_t uQ, uint32_t uK, uint32_t uV,
                                                    int qb, int S, int seq0, int head, int bh,
                                                    const DropoutRng& rng, int warp, int lane) {
  const int q4 = lane & 3;
  const float c = p.scale * 1.4426950408889634f;  // scale * log2(e)
  int qrow[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) qrow[e] = 64 * qb + 16 * warp + (lane >> 2) + 8 * e;

  float s[NB][32];
  wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < NB; ++kb)
#pragma unroll
    for (int k = 0; k < ATT_D / 16; ++k)
      Wgmma<64, kBF16, 0, 0>::ss(s[kb], gmma_desc(uQ + qb * SH_TILE + k * 32, 16, 1024),
                                 gmma_desc(uK + kb * SH_TILE + k * 32, 16, 1024), k != 0);
  wgmma_commit();
  wgmma_wait<0>();

  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int kb = 0; kb < NB; ++kb)
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int key = 64 * kb + 8 * (i >> 2) + 2 * q4 + (i & 1);
      if (key < S) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], s[kb][i]);
    }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    m[e] = fmaxf(m[e], __shfl_xor_sync(0xffffffffu, m[e], 1));
    m[e] = fmaxf(m[e], __shfl_xor_sync(0xffffffffu, m[e], 2));
  }
  const float mc[2] = {m[0] * c, m[1] * c};

  // probabilities in place of the scores: unnormalised exp(scale*(s - max)) in (0, 1]; O is
  // divided by the row sum at the end (the 1/l factor commutes with dropout and with P.V)
#pragma unroll
  for (int kb = 0; kb < NB; ++kb) {
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) {
      uint32_t dw[2][4];
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (p.drop_thr16) quad_drop_words(rng, bh, qrow[e], 64 * kb, jb, lane, dw[e]);
#pragma unroll
      for (int jq = 0; jq < 4; ++jq) {
        const int jj = 4 * jb + jq;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int i = 4 * jj + 2 * e + t;
            const int key = 64 * kb + 8 * jj + 2 * q4 + t;
            float pv = key < S ? ex2_approx(fmaf(s[kb][i], c, -mc[e])) : 0.f;
            l[e] += pv;
            if (p.drop_thr16) {
              // round P to 16 bit first (reference: softmax output is fp16, then dropout)
              const float pr = Elem<kBF16>::to_f(Elem<kBF16>::from_f(pv));
              pv = (rand16_half(dw[e][jq], t) < p.drop_thr16) ? 0.f : pr * p.drop_inv_keep;
            }
            s[kb][i] = pv;
          }
        }
      }
    }
  }

  float o[32];
  wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < NB; ++kb)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t a[4] = {Elem<kBF16>::pack(s[kb][8 * kk + 0], s[kb][8 * kk + 1]),
                             Elem<kBF16>::pack(s[kb][8 * kk + 2], s[kb][8 * kk + 3]),
                             Elem<kBF16>::pack(s[kb][8 * kk + 4], s[kb][8 * kk + 5]),
                             Elem<kBF16>::pack(s[kb][8 * kk + 6], s[kb][8 * kk + 7])};
      Wgmma<64, kBF16, 0, 1>::rs(o, a, gmma_desc(uV + kb * SH_TILE + kk * 2048, 8192, 1024), (kb | kk) != 0);
    }
  wgmma_commit();
  wgmma_wait<0>();

#pragma unroll
  for (int e = 0; e < 2; ++e) {
    l[e] += __shfl_xor_sync(0xffffffffu, l[e], 1);
    l[e] += __shfl_xor_sync(0xffffffffu, l[e], 2);
    if (qrow[e] >= S) continue;
    if (q4 == 0) p.lse[static_cast<size_t>(head) * p.T + seq0 + qrow[e]] = m[e] * p.scale + logf(l[e]);
    typename Elem<kBF16>::T* out = reinterpret_cast<typename Elem<kBF16>::T*>(p.ctx) +
                                   static_cast<size_t>(seq0 + qrow[e]) * p.H + head * ATT_D;
    store_frag_row<kBF16>(out, o, e, q4, 1.f / l[e]);
  }
}

template <bool kBF16>
__global__ void __launch_bounds__(SH_THREADS, 2)
attn_fwd_short_kernel(const __grid_constant__ CUtensorMap tmQKV64, const AttnParams p) {
  pdl_launch_dependents();
  pdl_wait();   // cu_seqlens / qkv come from preceding kernels
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                  // 2 slots each
  uint8_t* sK = smem + 2 * SH_TILE;
  uint8_t* sV = smem + 4 * SH_TILE;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 6 * SH_TILE);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV64);
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_barrier_init();
  }
  wg_sync();
  uint32_t rs0 = p.stream_lo, rs1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rs0, rs1);
  DropoutRng rng;
  rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = rs0; rng.s1 = rs1;

  auto load = [&](const ShortSched& it, int slot) {
    const int seq0 = p.cu_seqlens[it.b], nb = it.blocks(), col = it.h * ATT_D;
    mbar_expect_tx(&bar[slot], nb * 3 * SH_TILE);
    for (int r = 0; r < nb; ++r) {
      const int o = (slot + r) * SH_TILE;
      tma_load_2d(sQ + o, &tmQKV64, &bar[slot], col, seq0 + 64 * r);
      tma_load_2d(sK + o, &tmQKV64, &bar[slot], p.H + col, seq0 + 64 * r);
      tma_load_2d(sV + o, &tmQKV64, &bar[slot], 2 * p.H + col, seq0 + 64 * r);
    }
  };

  ShortSched it;
  it.init(p.cu_seqlens, p.B, p.nheads, lane);
  if (it.valid() && tid == 0) load(it, 0);
  int slot = 0;
  uint32_t ph = 0;   // bit s: parity of bar[s]
  while (it.valid()) {
    ShortSched nx = it;
    nx.next();
    const int seq0 = p.cu_seqlens[it.b], S = p.cu_seqlens[it.b + 1] - seq0, nb = it.blocks();
    const bool pre = nx.valid() && nb == 1 && nx.blocks() == 1;
    const int nslot = pre ? slot ^ 1 : 0;
    if (pre && tid == 0) load(nx, nslot);
    mbar_wait(&bar[slot], (ph >> slot) & 1);
    ph ^= 1u << slot;
    const uint32_t uQ = smem_u32(sQ + slot * SH_TILE), uK = smem_u32(sK + slot * SH_TILE),
                   uV = smem_u32(sV + slot * SH_TILE);
    const int bh = it.b * p.nheads + it.h;
    if (nb == 1) {
      attn_fwd_short_rows<kBF16, 1>(p, uQ, uK, uV, 0, S, seq0, it.h, bh, rng, warp, lane);
    } else {
#pragma unroll 1
      for (int qb = 0; qb < 2; ++qb)
        attn_fwd_short_rows<kBF16, 2>(p, uQ, uK, uV, qb, S, seq0, it.h, bh, rng, warp, lane);
    }
    wg_sync();   // every wgmma reading this stage has completed
    if (nx.valid() && !pre && tid == 0) load(nx, 0);
    it = nx;
    slot = nslot;
  }
}

constexpr int SH_FWD_SMEM = 6 * SH_TILE + 16 + 1024;

// dQ of query block qb = dS K : A = dS tiles [qb][0..NB), K-major over the item's keys;
// B = K [keys x d], MN-major
template <bool kBF16, int NB>
__device__ __forceinline__ void dq_block(float (&dq)[32], uint32_t uDS, uint32_t uK, int qb) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4 * NB; ++kk)
    Wgmma<64, kBF16, 0, 1>::ss(dq, gmma_desc(uDS + (qb * NB + (kk >> 2)) * SH_TILE + (kk & 3) * 32, 16, 1024),
                               gmma_desc(uK + kk * 2048, 8192, 1024), kk != 0);
  wgmma_commit();
  wgmma_wait<0>();
}

// kBias = false: the deterministic mode's instantiation, with no bias-gradient flush (its float atomics);
// that mode sums the bias gradient from dqkv with launch_colsum_det instead.
template <bool kBF16, bool kBias = true>
__global__ void __launch_bounds__(SH_THREADS, 2)
attn_bwd_short_kernel(const __grid_constant__ CUtensorMap tmQKV64, const __grid_constant__ CUtensorMap tmDO64,
                      const AttnParams p) {
  using T16 = typename Elem<kBF16>::T;
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // this CTA's partial QKV bias gradient of the current head, one [q | k | v] x 64 slice per warp
  __shared__ float sBias[4][3 * ATT_D];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                   // 2 slots each
  uint8_t* sK = smem + 2 * SH_TILE;
  uint8_t* sV = smem + 4 * SH_TILE;
  uint8_t* sdO = smem + 6 * SH_TILE;
  uint8_t* sP = smem + 8 * SH_TILE;     // Pd of one (query block, key block)
  uint8_t* sDS = smem + 9 * SH_TILE;    // dS, tile [qb][kb] at (qb * nb + kb) * SH_TILE
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 13 * SH_TILE);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q4 = lane & 3;
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV64);
    tma_prefetch_desc(&tmDO64);
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_barrier_init();
  }
  for (int i = tid; i < 4 * 3 * ATT_D; i += SH_THREADS) (&sBias[0][0])[i] = 0.f;
  wg_sync();
  uint32_t rs0 = p.stream_lo, rs1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rs0, rs1);
  DropoutRng rng;
  rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = rs0; rng.s1 = rs1;
  const float c = p.scale * 1.4426950408889634f;
  int r_loc[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) r_loc[e] = 16 * warp + (lane >> 2) + 8 * e;
  const uint32_t uP = smem_u32(sP), uDS = smem_u32(sDS);

  auto load = [&](const ShortSched& it, int slot) {
    const int seq0 = p.cu_seqlens[it.b], nb = it.blocks(), col = it.h * ATT_D;
    mbar_expect_tx(&bar[slot], nb * 4 * SH_TILE);
    for (int r = 0; r < nb; ++r) {
      const int o = (slot + r) * SH_TILE;
      tma_load_2d(sQ + o, &tmQKV64, &bar[slot], col, seq0 + 64 * r);
      tma_load_2d(sK + o, &tmQKV64, &bar[slot], p.H + col, seq0 + 64 * r);
      tma_load_2d(sV + o, &tmQKV64, &bar[slot], 2 * p.H + col, seq0 + 64 * r);
      tma_load_2d(sdO + o, &tmDO64, &bar[slot], col, seq0 + 64 * r);
    }
  };

  ShortSched it;
  it.init(p.cu_seqlens, p.B, p.nheads, lane);
  if (it.valid() && tid == 0) load(it, 0);
  int slot = 0;
  uint32_t ph = 0;   // bit s: parity of bar[s]
  while (it.valid()) {
    ShortSched nx = it;
    nx.next();
    const int seq0 = p.cu_seqlens[it.b], S = p.cu_seqlens[it.b + 1] - seq0, nb = it.blocks();
    const int head = it.h, bh = it.b * p.nheads + head;
    const bool pre = nx.valid() && nb == 1 && nx.blocks() == 1;
    const int nslot = pre ? slot ^ 1 : 0;
    if (pre && tid == 0) load(nx, nslot);
    mbar_wait(&bar[slot], (ph >> slot) & 1);
    ph ^= 1u << slot;
    const uint32_t uQ = smem_u32(sQ + slot * SH_TILE), udO = smem_u32(sdO + slot * SH_TILE),
                   uK = smem_u32(sK + slot * SH_TILE), uV = smem_u32(sV + slot * SH_TILE);

    for (int kb = 0; kb < nb; ++kb) {
      float dv[32], dk[32];
      for (int qb = 0; qb < nb; ++qb) {
        int qrow[2];
        bool q_ok[2];
        float delta[2], lse2[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          qrow[e] = 64 * qb + r_loc[e];
          q_ok[e] = qrow[e] < S;
          row_delta_lse<kBF16>(p, seq0, head, qrow[e], q_ok[e], q4, delta[e], lse2[e]);
        }
        float s[32], dp[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < ATT_D / 16; ++k)   // S = Q K^T
          Wgmma<64, kBF16, 0, 0>::ss(s, gmma_desc(uQ + qb * SH_TILE + k * 32, 16, 1024),
                                     gmma_desc(uK + kb * SH_TILE + k * 32, 16, 1024), k != 0);
#pragma unroll
        for (int k = 0; k < ATT_D / 16; ++k)   // dPd = dO V^T
          Wgmma<64, kBF16, 0, 0>::ss(dp, gmma_desc(udO + qb * SH_TILE + k * 32, 16, 1024),
                                     gmma_desc(uV + kb * SH_TILE + k * 32, 16, 1024), k != 0);
        wgmma_commit();
        wgmma_wait<0>();

        uint8_t* dsTile = sDS + (qb * nb + kb) * SH_TILE;
#pragma unroll
        for (int jb = 0; jb < 2; ++jb) {
          uint32_t dw[2][4];
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (p.drop_thr16) quad_drop_words(rng, bh, qrow[e], 64 * kb, jb, lane, dw[e]);
#pragma unroll
          for (int jq = 0; jq < 4; ++jq) {
            const int jj = 4 * jb + jq;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float pd[2], ds[2];
#pragma unroll
              for (int t = 0; t < 2; ++t) {
                const int idx = 4 * jj + 2 * e + t;
                const bool ok = q_ok[e] && 64 * kb + 8 * jj + 2 * q4 + t < S;
                float pr = ok ? ex2_approx(fmaf(s[idx], c, -lse2[e])) : 0.f;
                pr = Elem<kBF16>::to_f(Elem<kBF16>::from_f(pr));   // P as the forward rounded it
                float dpv = dp[idx];
                float pdv = pr;
                if (p.drop_thr16) {
                  const bool drop = rand16_half(dw[e][jq], t) < p.drop_thr16;
                  pdv = drop ? 0.f : pr * p.drop_inv_keep;
                  dpv = drop ? 0.f : dpv * p.drop_inv_keep;
                }
                pd[t] = pdv;
                ds[t] = ok ? pr * (dpv - delta[e]) * p.scale : 0.f;
              }
              st_swz128_u32(sP, r_loc[e], 8 * jj + 2 * q4, Elem<kBF16>::pack(pd[0], pd[1]));
              st_swz128_u32(dsTile, r_loc[e], 8 * jj + 2 * q4, Elem<kBF16>::pack(ds[0], ds[1]));
            }
          }
        }
        fence_proxy_async_smem();
        wg_sync();

        // dV += Pd^T dO ; dK += dS^T Q : A = [queries x keys] read MN-major (M = the 64 keys of
        // block kb), B = [queries x d] read MN-major (N = d); contraction over the 64 queries of qb.
        const uint32_t uDSt = smem_u32(dsTile);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          Wgmma<64, kBF16, 1, 1>::ss(dv, gmma_desc(uP + kk * 2048, SH_TILE, 1024),
                                     gmma_desc(udO + qb * SH_TILE + kk * 2048, 8192, 1024), (qb | kk) != 0);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          Wgmma<64, kBF16, 1, 1>::ss(dk, gmma_desc(uDSt + kk * 2048, SH_TILE, 1024),
                                     gmma_desc(uQ + qb * SH_TILE + kk * 2048, 8192, 1024), (qb | kk) != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wg_sync();   // sP is rewritten by the next (qb, kb)
      }
      // dK, dV of key block kb out (rows = keys)
      int key[2];
      bool k_ok[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        key[e] = 64 * kb + r_loc[e];
        k_ok[e] = key[e] < S;
      }
      if (kBias && p.dbias) {   // key / value bias gradients
        frag_colsum64_warp(dk, k_ok[0], k_ok[1], sBias[warp] + ATT_D, lane);
        frag_colsum64_warp(dv, k_ok[0], k_ok[1], sBias[warp] + 2 * ATT_D, lane);
      }
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (!k_ok[e]) continue;
        T16* outk = reinterpret_cast<T16*>(p.dqkv) + static_cast<size_t>(seq0 + key[e]) * (3 * p.H) + p.H +
                    head * ATT_D;
        store_frag_row<kBF16>(outk, dk, e, q4, 1.f);
        store_frag_row<kBF16>(outk + p.H, dv, e, q4, 1.f);
      }
    }

    for (int qb = 0; qb < nb; ++qb) {
      float dq[32];
      if (nb == 1) dq_block<kBF16, 1>(dq, uDS, uK, 0);
      else dq_block<kBF16, 2>(dq, uDS, uK, qb);
      bool q_ok[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) q_ok[e] = 64 * qb + r_loc[e] < S;
      if (kBias && p.dbias) frag_colsum64_warp(dq, q_ok[0], q_ok[1], sBias[warp], lane);   // query-bias gradient
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (q_ok[e])
          store_frag_row<kBF16>(reinterpret_cast<T16*>(p.dqkv) + static_cast<size_t>(seq0 + 64 * qb + r_loc[e]) *
                                                                       (3 * p.H) + head * ATT_D,
                                dq, e, q4, 1.f);
    }
    wg_sync();   // every wgmma reading this stage, sP and sDS has completed; sBias is complete
    if (nx.valid() && !pre && tid == 0) load(nx, 0);
    if (kBias && p.dbias && (!nx.valid() || nx.h != head)) {
      // one atomic per column and head change: this CTA's share of the bias gradient of `head`
      for (int i = tid; i < 3 * ATT_D; i += SH_THREADS) {
        atomicAdd(p.dbias + (i >> 6) * p.H + head * ATT_D + (i & 63),
                  (sBias[0][i] + sBias[1][i]) + (sBias[2][i] + sBias[3][i]));
        sBias[0][i] = sBias[1][i] = sBias[2][i] = sBias[3][i] = 0.f;
      }
      // the next writes to sBias follow the next item's first wg_sync
    }
    it = nx;
    slot = nslot;
  }
}

constexpr int SH_BWD_SMEM = 13 * SH_TILE + 16 + 1024;

// S[64 rows of warpgroup wg, 128 keys] = A[rows] . B[keys]^T, both K-major 128 x 64 tiles
template <bool kBF16>
__device__ __forceinline__ void qk_block(float (&s)[64], uint32_t sA, uint32_t sB, int wg) {
#pragma unroll
  for (int k = 0; k < ATT_D / 16; ++k)
    Wgmma<128, kBF16, 0, 0>::ss(s, gmma_desc(sA + wg * (64 * 128) + k * 32, 16, 1024),
                                gmma_desc(sB + k * 32, 16, 1024), k != 0);
}

// =====================================================================================
// Long sequences (max_seqlen > 128).  One CTA per (128-query tile, head, sequence): two
// warpgroups, each owning 64 query rows; two sweeps over 128-key blocks (row max, then P and
// O = P V).
// =====================================================================================
template <bool kBF16>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const AttnParams p) {
  pdl_launch_dependents();
  pdl_wait();   // cu_seqlens / qkv come from preceding kernels
  const int b = blockIdx.z, qt = blockIdx.x;
  const int seq0 = p.cu_seqlens[b];
  const int S = p.cu_seqlens[b + 1] - seq0;
  if (qt * ATT_BM >= S) return;  // whole CTA exits together, before any barrier use
  const int head = blockIdx.y;
  const int nkv = (S + ATT_BN - 1) / ATT_BN;
  uint32_t rs0 = p.stream_lo, rs1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rs0, rs1);

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_TILE;
  uint8_t* sV = smem + 2 * ATT_TILE;
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + 3 * ATT_TILE);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, q4 = lane & 3;
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV);
    mbar_init(bar_load, 1);
    fence_barrier_init();
  }
  __syncthreads();

  // this thread's two query rows
  int qrow[2];
  bool q_ok[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    qrow[e] = qt * ATT_BM + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * e;
    q_ok[e] = qrow[e] < S;
  }
  const int bh = b * p.nheads + head;
  const float c = p.scale * 1.4426950408889634f;  // scale * log2(e)
  const uint32_t uQ = smem_u32(sQ), uK = smem_u32(sK), uV = smem_u32(sV);
  uint32_t ph_load = 0;
  float s[64];

  // ---------------------------------------------------------------- sweep 1: row max
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  for (int j = 0; j < nkv; ++j) {
    const int kv_len = min(ATT_BN, S - j * ATT_BN);
    if (tid == 0) {
      const bool with_v = (nkv == 1);
      mbar_expect_tx(bar_load, (j == 0 ? ATT_TILE : 0) + ATT_TILE + (with_v ? ATT_TILE : 0));
      if (j == 0) tma_load_2d(sQ, &tmQKV, bar_load, head * ATT_D, seq0 + qt * ATT_BM);
      tma_load_2d(sK, &tmQKV, bar_load, p.H + head * ATT_D, seq0 + j * ATT_BN);
      if (with_v) tma_load_2d(sV, &tmQKV, bar_load, 2 * p.H + head * ATT_D, seq0 + j * ATT_BN);
    }
    mbar_wait(bar_load, ph_load);
    ph_load ^= 1;
    wgmma_fence();
    qk_block<kBF16>(s, uQ, uK, wg);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int key = 8 * (i >> 2) + 2 * q4 + (i & 1);
      if (key < kv_len) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], s[i]);
    }
    if (nkv > 1) __syncthreads();   // sK is about to be overwritten
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    m[e] = fmaxf(m[e], __shfl_xor_sync(0xffffffffu, m[e], 1));
    m[e] = fmaxf(m[e], __shfl_xor_sync(0xffffffffu, m[e], 2));
  }
  const float mc[2] = {m[0] * c, m[1] * c};

  // ---------------------------------------------------------------- sweep 2: P and O = P V
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  for (int j = 0; j < nkv; ++j) {
    const int kv_len = min(ATT_BN, S - j * ATT_BN);
    if (nkv > 1) {
      if (tid == 0) {
        mbar_expect_tx(bar_load, 2 * ATT_TILE);
        tma_load_2d(sK, &tmQKV, bar_load, p.H + head * ATT_D, seq0 + j * ATT_BN);
        tma_load_2d(sV, &tmQKV, bar_load, 2 * p.H + head * ATT_D, seq0 + j * ATT_BN);
      }
      mbar_wait(bar_load, ph_load);
      ph_load ^= 1;
      wgmma_fence();
      qk_block<kBF16>(s, uQ, uK, wg);
      wgmma_commit();
      wgmma_wait<0>();
    }
    // probabilities in place of the scores: unnormalised exp(scale*(s - max)) in (0, 1]; O is
    // divided by the row sum at the end (the 1/l factor commutes with dropout and with P.V)
    DropoutRng rng;
    rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = rs0; rng.s1 = rs1;
#pragma unroll
    for (int jb = 0; jb < 4; ++jb) {
      uint32_t dw[2][4];
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (p.drop_thr16) quad_drop_words(rng, bh, qrow[e], j * ATT_BN, jb, lane, dw[e]);
#pragma unroll
      for (int jq = 0; jq < 4; ++jq) {
        const int jj = 4 * jb + jq;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int i = 4 * jj + 2 * e + t;
            const int key = 8 * jj + 2 * q4 + t;
            float pv = key < kv_len ? ex2_approx(fmaf(s[i], c, -mc[e])) : 0.f;
            l[e] += pv;
            if (p.drop_thr16) {
              // round P to 16 bit first (reference: softmax output is fp16, then dropout)
              const float pr = Elem<kBF16>::to_f(Elem<kBF16>::from_f(pv));
              pv = (rand16_half(dw[e][jq], t) < p.drop_thr16) ? 0.f : pr * p.drop_inv_keep;
            }
            s[i] = pv;
          }
        }
      }
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) {
      const uint32_t a[4] = {Elem<kBF16>::pack(s[8 * kk + 0], s[8 * kk + 1]),
                             Elem<kBF16>::pack(s[8 * kk + 2], s[8 * kk + 3]),
                             Elem<kBF16>::pack(s[8 * kk + 4], s[8 * kk + 5]),
                             Elem<kBF16>::pack(s[8 * kk + 6], s[8 * kk + 7])};
      Wgmma<64, kBF16, 0, 1>::rs(o, a, gmma_desc(uV + kk * 2048, 8192, 1024), (j | kk) != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (nkv > 1) __syncthreads();   // sK / sV are about to be overwritten
  }

  // ---------------------------------------------------------------- epilogue: O / l -> ctx[T, H]
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    l[e] += __shfl_xor_sync(0xffffffffu, l[e], 1);
    l[e] += __shfl_xor_sync(0xffffffffu, l[e], 2);
    if (!q_ok[e]) continue;
    if (q4 == 0) p.lse[static_cast<size_t>(head) * p.T + seq0 + qrow[e]] = m[e] * p.scale + logf(l[e]);
    typename Elem<kBF16>::T* out = reinterpret_cast<typename Elem<kBF16>::T*>(p.ctx) +
                                   static_cast<size_t>(seq0 + qrow[e]) * p.H + head * ATT_D;
    store_frag_row<kBF16>(out, o, e, q4, 1.f / l[e]);
  }
}

constexpr int ATT_FWD_SMEM = 3 * ATT_TILE + 64 + 1024;

// =====================================================================================
// Backward, long sequences.  One CTA per (128-key block j, head, sequence); loops over 128-query
// blocks i.
//   smem: Q_i, dO_i, K_j, V_j (TMA, 128B swizzle) + Pd and dS written by the softmax threads
//   (row = query, 64-key slabs) and consumed both K-major (dQ = dS K) and MN-major
//   (dV = Pd^T dO, dK = dS^T Q) by wgmma.  Warpgroup wg owns query rows [64 wg, +64) of S / dP /
//   dQ and key rows [64 wg, +64) of dK / dV (the accumulators of dK / dV live across the loop).
// dQ of a sequence longer than one key block is accumulated with fp32 atomics in `dq_accum`.
// =====================================================================================
template <bool kBF16>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO,
                const AttnParams p, float* dq_accum) {
  using T16 = typename Elem<kBF16>::T;
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.z, j = blockIdx.x;
  const int seq0 = p.cu_seqlens[b];
  const int S = p.cu_seqlens[b + 1] - seq0;
  if (j * ATT_BN >= S) return;
  const int head = blockIdx.y;
  const int nq = (S + ATT_BM - 1) / ATT_BM;
  const int nkv = (S + ATT_BN - 1) / ATT_BN;
  uint32_t rs0 = p.stream_lo, rs1 = p.stream_hi;
  if (p.drop_thr16) rng_add_dev_offset(p.rng_dev, rs0, rs1);
  const int kv_len = min(ATT_BN, S - j * ATT_BN);

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sdO = smem + ATT_TILE;
  uint8_t* sK = smem + 2 * ATT_TILE;
  uint8_t* sV = smem + 3 * ATT_TILE;
  uint8_t* sP = smem + 4 * ATT_TILE;    // 2 slabs
  uint8_t* sDS = smem + 6 * ATT_TILE;   // 2 slabs
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(smem + 8 * ATT_TILE);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2, q4 = lane & 3;
  if (tid == 0) {
    tma_prefetch_desc(&tmQKV);
    tma_prefetch_desc(&tmDO);
    mbar_init(bar_load, 1);
    fence_barrier_init();
  }
  __syncthreads();
  int r_loc[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) r_loc[e] = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * e;
  const int bh = b * p.nheads + head;
  const float c = p.scale * 1.4426950408889634f;
  const uint32_t uQ = smem_u32(sQ), udO = smem_u32(sdO), uK = smem_u32(sK), uV = smem_u32(sV);
  const uint32_t uP = smem_u32(sP), uDS = smem_u32(sDS);
  uint32_t ph_load = 0;
  float dv[32], dk[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) { dv[i] = 0.f; dk[i] = 0.f; }

  for (int i = 0; i < nq; ++i) {
    int qrow[2];
    bool q_ok[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      qrow[e] = i * ATT_BM + r_loc[e];
      q_ok[e] = qrow[e] < S;
    }
    if (tid == 0) {
      mbar_expect_tx(bar_load, (i == 0 ? 4 : 2) * ATT_TILE);
      tma_load_2d(sQ, &tmQKV, bar_load, head * ATT_D, seq0 + i * ATT_BM);
      tma_load_2d(sdO, &tmDO, bar_load, head * ATT_D, seq0 + i * ATT_BM);
      if (i == 0) {
        tma_load_2d(sK, &tmQKV, bar_load, p.H + head * ATT_D, seq0 + j * ATT_BN);
        tma_load_2d(sV, &tmQKV, bar_load, 2 * p.H + head * ATT_D, seq0 + j * ATT_BN);
      }
    }

    // delta and the saved log-sum-exp, straight from global (overlaps the loads)
    float delta[2], lse2[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) row_delta_lse<kBF16>(p, seq0, head, qrow[e], q_ok[e], q4, delta[e], lse2[e]);

    mbar_wait(bar_load, ph_load);
    ph_load ^= 1;
    float s[64], dp[64];
    wgmma_fence();
    qk_block<kBF16>(s, uQ, uK, wg);     // S = Q K^T
    qk_block<kBF16>(dp, udO, uV, wg);   // dPd = dO V^T
    wgmma_commit();
    wgmma_wait<0>();

    DropoutRng rng;
    rng.k0 = p.seed_lo; rng.k1 = p.seed_hi; rng.s0 = rs0; rng.s1 = rs1;
#pragma unroll
    for (int jb = 0; jb < 4; ++jb) {
      uint32_t dw[2][4];
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (p.drop_thr16) quad_drop_words(rng, bh, qrow[e], j * ATT_BN, jb, lane, dw[e]);
#pragma unroll
      for (int jq = 0; jq < 4; ++jq) {
        const int jj = 4 * jb + jq;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float pd[2], ds[2];
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int idx = 4 * jj + 2 * e + t;
            const int key = 8 * jj + 2 * q4 + t;
            const bool ok = q_ok[e] && key < kv_len;
            float pr = ok ? ex2_approx(fmaf(s[idx], c, -lse2[e])) : 0.f;
            pr = Elem<kBF16>::to_f(Elem<kBF16>::from_f(pr));   // P as the forward rounded it
            float dpv = dp[idx];
            float pdv = pr;
            if (p.drop_thr16) {
              const bool drop = rand16_half(dw[e][jq], t) < p.drop_thr16;
              pdv = drop ? 0.f : pr * p.drop_inv_keep;
              dpv = drop ? 0.f : dpv * p.drop_inv_keep;
            }
            pd[t] = pdv;
            ds[t] = ok ? pr * (dpv - delta[e]) * p.scale : 0.f;
          }
          st_swz128_u32(sP, r_loc[e], 8 * jj + 2 * q4, Elem<kBF16>::pack(pd[0], pd[1]));
          st_swz128_u32(sDS, r_loc[e], 8 * jj + 2 * q4, Elem<kBF16>::pack(ds[0], ds[1]));
        }
      }
    }
    fence_proxy_async_smem();
    __syncthreads();

    float dq[32];
    wgmma_fence();
    // dV += Pd^T dO ; dK += dS^T Q : A = [queries x keys] read MN-major (M = keys of this
    // warpgroup = slab wg), B = [queries x d] read MN-major (N = d); contraction over 128 queries.
#pragma unroll
    for (int kk = 0; kk < ATT_BM / 16; ++kk)
      Wgmma<64, kBF16, 1, 1>::ss(dv, gmma_desc(uP + wg * ATT_TILE + kk * 2048, ATT_TILE, 1024),
                                 gmma_desc(udO + kk * 2048, 8192, 1024), (i | kk) != 0);
#pragma unroll
    for (int kk = 0; kk < ATT_BM / 16; ++kk)
      Wgmma<64, kBF16, 1, 1>::ss(dk, gmma_desc(uDS + wg * ATT_TILE + kk * 2048, ATT_TILE, 1024),
                                 gmma_desc(uQ + kk * 2048, 8192, 1024), (i | kk) != 0);
    // dQ = dS K : A K-major over keys (rows = this warpgroup's queries), B = K_j [keys x d] MN-major
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk)
      Wgmma<64, kBF16, 0, 1>::ss(dq, gmma_desc(uDS + (kk >> 2) * ATT_TILE + wg * (64 * 128) + (kk & 3) * 32, 16, 1024),
                                 gmma_desc(uK + kk * 2048, 8192, 1024), kk != 0);
    wgmma_commit();
    wgmma_wait<0>();
    if (p.dbias)   // query-bias gradient: this key block's share of colsum(dQ) for `head`
      frag_colsum64_atomic(dq, q_ok[0], q_ok[1], p.dbias + head * ATT_D, lane);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if (!q_ok[e]) continue;
      if (nkv == 1) {
        store_frag_row<kBF16>(reinterpret_cast<T16*>(p.dqkv) + static_cast<size_t>(seq0 + qrow[e]) * (3 * p.H) +
                                  head * ATT_D, dq, e, q4, 1.f);
      } else {
        float* acc = dq_accum + static_cast<size_t>(seq0 + qrow[e]) * p.H + head * ATT_D;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          atomicAdd(acc + 8 * jj + 2 * q4, dq[4 * jj + 2 * e]);
          atomicAdd(acc + 8 * jj + 2 * q4 + 1, dq[4 * jj + 2 * e + 1]);
        }
      }
    }
    if (i + 1 < nq) __syncthreads();   // next iteration overwrites sQ / sdO / sP / sDS
  }

  // dK_j, dV_j out (rows = keys)
  int key[2];
  bool k_ok[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    key[e] = j * ATT_BN + r_loc[e];
    k_ok[e] = key[e] < S;
  }
  if (p.dbias) {   // key / value bias gradients
    frag_colsum64_atomic(dk, k_ok[0], k_ok[1], p.dbias + p.H + head * ATT_D, lane);
    frag_colsum64_atomic(dv, k_ok[0], k_ok[1], p.dbias + 2 * p.H + head * ATT_D, lane);
  }
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    if (!k_ok[e]) continue;
    T16* outk = reinterpret_cast<T16*>(p.dqkv) + static_cast<size_t>(seq0 + key[e]) * (3 * p.H) + p.H +
                head * ATT_D;
    store_frag_row<kBF16>(outk, dk, e, q4, 1.f);
    store_frag_row<kBF16>(outk + p.H, dv, e, q4, 1.f);
  }
}

// dqkv[:, 0:H] (16-bit) = dq_accum (fp32) for sequences spanning several key blocks (others
// wrote dQ directly).  One CTA per sequence.
template <bool kBF16>
__global__ void attn_dq_convert_kernel(const float* __restrict__ acc, void* dqkv,
                                       const int* __restrict__ cu_seqlens, int H) {
  pdl_launch_dependents();
  pdl_wait();
  const int seq0 = cu_seqlens[blockIdx.x];
  const int S = cu_seqlens[blockIdx.x + 1] - seq0;
  if (S <= ATT_BN) return;
  const int nvec = S * H / 8;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    const int row = (v * 8) / H, col = (v * 8) % H;
    const float* src = acc + static_cast<size_t>(seq0 + row) * H + col;
    const float4 a = *reinterpret_cast<const float4*>(src);
    const float4 b = *reinterpret_cast<const float4*>(src + 4);
    uint4 u;
    u.x = Elem<kBF16>::pack(a.x, a.y); u.y = Elem<kBF16>::pack(a.z, a.w);
    u.z = Elem<kBF16>::pack(b.x, b.y); u.w = Elem<kBF16>::pack(b.z, b.w);
    *reinterpret_cast<uint4*>(reinterpret_cast<typename Elem<kBF16>::T*>(dqkv) +
                              static_cast<size_t>(seq0 + row) * 3 * H + col) = u;
  }
}

constexpr int ATT_BWD_SMEM = 8 * ATT_TILE + 64 + 1024;

// Parameters shared by forward and backward.
static AttnParams attn_params(const ub200_attn_args& a) {
  AttnParams p{};
  p.cu_seqlens = a.cu_seqlens;
  p.B = a.batch; p.H = a.hidden; p.nheads = a.num_heads; p.T = a.total_tokens;
  p.ctx = a.ctx; p.lse = a.lse;
  p.scale = 0.125f;
  if (a.dropout_p > 0.f) {
    const DropoutThreshold d = dropout_threshold(a.dropout_p);
    p.drop_thr16 = d.thr16;
    p.drop_inv_keep = d.inv_keep;
  } else {
    p.drop_thr16 = 0; p.drop_inv_keep = 1.f;
  }
  p.seed_lo = static_cast<uint32_t>(a.rng_seed); p.seed_hi = static_cast<uint32_t>(a.rng_seed >> 32);
  p.stream_lo = static_cast<uint32_t>(a.rng_stream);
  p.stream_hi = static_cast<uint32_t>(a.rng_stream >> 32);
  p.rng_dev = reinterpret_cast<const unsigned long long*>(a.rng_offset_dev);
  return p;
}

// persistent grid of the short kernels: `per_sm` CTAs on every SM, no more than there are items
static dim3 short_grid(const ub200_attn_args& a, int per_sm) {
  const long long items = static_cast<long long>(a.batch) * a.num_heads;
  const long long g = static_cast<long long>(num_sms()) * per_sm;
  return dim3(static_cast<unsigned>(g < items ? g : items));
}

}  // namespace ub

extern "C" int ub200_attn_fwd(const ub200_attn_args* args, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(args != nullptr, "attn_fwd: args is NULL");
  const ub200_attn_args& a = *args;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  UB_CHECK_ARG(a.qkv && a.ctx && a.lse && a.cu_seqlens, "attn_fwd: null pointer");
  UB_CHECK_ARG(a.batch > 0 && a.total_tokens > 0, "attn_fwd: empty batch");
  UB_CHECK_ARG(a.num_heads > 0 && a.hidden == a.num_heads * ATT_D,
               "attn_fwd: head_dim must be 64 (hidden=%d heads=%d)", a.hidden, a.num_heads);
  UB_CHECK_ARG(a.max_seqlen > 0 && a.max_seqlen <= ATT_MAXSEQ,
               "attn_fwd: max_seqlen %d outside (0, %d]", a.max_seqlen, ATT_MAXSEQ);
  UB_CHECK_ARG(a.dtype == UB200_F16 || a.dtype == UB200_BF16, "attn_fwd: bad dtype");
  UB_CHECK_ARG(a.dropout_p >= 0.f && a.dropout_p < 1.f, "attn_fwd: dropout_p out of range");

  const AttnParams p = attn_params(a);
  const bool bf = a.dtype == UB200_BF16;
  CUtensorMap tm;
  if (a.max_seqlen <= SH_MAXSEQ) {
    int rc = make_tma_2d(&tm, a.qkv, a.dtype, a.total_tokens, 3 * a.hidden, 3 * a.hidden, 64, ATT_D);
    if (rc) return rc;
    void (*kern)(const CUtensorMap, const AttnParams) = bf ? attn_fwd_short_kernel<true> : attn_fwd_short_kernel<false>;
    static unsigned long long configured[2] = {0, 0};   // one bit per device
    if (first_use_on_device(configured[bf ? 1 : 0]))
      UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_FWD_SMEM));
    ProfScope ps(stream);
    UB_CHECK_CUDA(launch_pdl(kern, short_grid(a, 2), dim3(SH_THREADS), SH_FWD_SMEM, stream, 1, tm, p));
  } else {
    int rc = make_tma_2d(&tm, a.qkv, a.dtype, a.total_tokens, 3 * a.hidden, 3 * a.hidden, ATT_BM, ATT_D);
    if (rc) return rc;
    dim3 grid((a.max_seqlen + ATT_BM - 1) / ATT_BM, a.num_heads, a.batch);
    void (*kern)(const CUtensorMap, const AttnParams) = bf ? attn_fwd_kernel<true> : attn_fwd_kernel<false>;
    static unsigned long long configured[2] = {0, 0};   // one bit per device
    if (first_use_on_device(configured[bf ? 1 : 0]))
      UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_FWD_SMEM));
    ProfScope ps(stream);
    UB_CHECK_CUDA(launch_pdl(kern, grid, dim3(ATT_THREADS), ATT_FWD_SMEM, stream, 1, tm, p));
  }
  UB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int64_t ub200_attn_bwd_workspace_bytes(int32_t total_tokens, int32_t hidden,
                                                  int32_t max_seqlen) {
  // fp32 dQ accumulator, only touched when some sequence is longer than one 128-key block
  if (max_seqlen <= ub::ATT_BN) return 0;
  return static_cast<int64_t>(total_tokens) * hidden * 4;
}

extern "C" int ub200_attn_bwd(const ub200_attn_args* args, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(args != nullptr, "attn_bwd: args is NULL");
  const ub200_attn_args& a = *args;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  UB_CHECK_ARG(a.qkv && a.ctx && a.lse && a.cu_seqlens && a.dctx && a.dqkv, "attn_bwd: null pointer");
  UB_CHECK_ARG(a.batch > 0 && a.total_tokens > 0, "attn_bwd: empty batch");
  UB_CHECK_ARG(a.num_heads > 0 && a.hidden == a.num_heads * ATT_D, "attn_bwd: head_dim must be 64");
  UB_CHECK_ARG(a.max_seqlen > 0 && a.max_seqlen <= ATT_MAXSEQ, "attn_bwd: max_seqlen %d outside (0, %d]",
               a.max_seqlen, ATT_MAXSEQ);
  UB_CHECK_ARG(a.dtype == UB200_F16 || a.dtype == UB200_BF16, "attn_bwd: bad dtype");
  const bool multi = a.max_seqlen > ATT_BN;
  UB_CHECK_ARG(!multi || a.workspace, "attn_bwd: max_seqlen > 128 needs the dQ workspace");

  AttnParams p = attn_params(a);
  p.dctx = a.dctx; p.dqkv = a.dqkv; p.dbias = a.dbias;
  const int di = a.dtype == UB200_BF16 ? 1 : 0;

  if (deterministic()) {
    // dQ of a sequence longer than one key block is summed over key blocks with float atomics; no
    // fixed-order form of the long kernels exists yet
    if (a.max_seqlen > SH_MAXSEQ)
      return set_error(UB200_EUNSUPPORTED, "attn_bwd: deterministic mode supports max_seqlen <= %d (got %d)",
                       SH_MAXSEQ, a.max_seqlen);
    CUtensorMap tmQ, tmD;
    int rc = make_tma_2d(&tmQ, a.qkv, a.dtype, a.total_tokens, 3 * a.hidden, 3 * a.hidden, 64, ATT_D);
    if (rc) return rc;
    rc = make_tma_2d(&tmD, a.dctx, a.dtype, a.total_tokens, a.hidden, a.hidden, 64, ATT_D);
    if (rc) return rc;
    p.dbias = nullptr;
    void (*kern)(const CUtensorMap, const CUtensorMap, const AttnParams) =
        di ? attn_bwd_short_kernel<true, false> : attn_bwd_short_kernel<false, false>;
    static unsigned long long configured[2] = {0, 0};   // one bit per device
    if (first_use_on_device(configured[di]))
      UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_BWD_SMEM));
    {
      ProfScope ps(stream);
      UB_CHECK_CUDA(launch_pdl(kern, short_grid(a, 2), dim3(SH_THREADS), SH_BWD_SMEM, stream, 1, tmQ, tmD, p));
    }
    UB_CHECK_CUDA(cudaGetLastError());
    // QKV bias gradient: fixed-order column sums of the 16-bit dqkv, over the rows of the sequences only
    // (rows past cu_seqlens[batch] are not written by the kernel)
    if (a.dbias)
      return launch_colsum_det(a.dtype, a.dqkv, a.dbias, a.total_tokens, 3 * a.hidden, 3 * a.hidden, stream,
                               a.cu_seqlens + a.batch);
    return 0;
  }

  if (a.max_seqlen <= SH_MAXSEQ) {
    CUtensorMap tmQ, tmD;
    int rc = make_tma_2d(&tmQ, a.qkv, a.dtype, a.total_tokens, 3 * a.hidden, 3 * a.hidden, 64, ATT_D);
    if (rc) return rc;
    rc = make_tma_2d(&tmD, a.dctx, a.dtype, a.total_tokens, a.hidden, a.hidden, 64, ATT_D);
    if (rc) return rc;
    void (*kern)(const CUtensorMap, const CUtensorMap, const AttnParams) =
        di ? attn_bwd_short_kernel<true> : attn_bwd_short_kernel<false>;
    static unsigned long long configured[2] = {0, 0};   // one bit per device
    if (first_use_on_device(configured[di]))
      UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SH_BWD_SMEM));
    ProfScope ps(stream);
    UB_CHECK_CUDA(launch_pdl(kern, short_grid(a, 2), dim3(SH_THREADS), SH_BWD_SMEM, stream, 1, tmQ, tmD, p));
    UB_CHECK_CUDA(cudaGetLastError());
    return 0;
  }

  CUtensorMap tmQ, tmD;
  int rc = make_tma_2d(&tmQ, a.qkv, a.dtype, a.total_tokens, 3 * a.hidden, 3 * a.hidden, ATT_BM, ATT_D);
  if (rc) return rc;
  rc = make_tma_2d(&tmD, a.dctx, a.dtype, a.total_tokens, a.hidden, a.hidden, ATT_BM, ATT_D);
  if (rc) return rc;
  float* acc = reinterpret_cast<float*>(a.workspace);
  UB_CHECK_CUDA(cudaMemsetAsync(acc, 0, static_cast<size_t>(a.total_tokens) * a.hidden * 4, stream));

  dim3 grid((a.max_seqlen + ATT_BN - 1) / ATT_BN, a.num_heads, a.batch);
  void (*kern)(const CUtensorMap, const CUtensorMap, const AttnParams, float*) =
      di ? attn_bwd_kernel<true> : attn_bwd_kernel<false>;
  static unsigned long long configured[2] = {0, 0};   // one bit per device
  if (first_use_on_device(configured[di]))
    UB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_BWD_SMEM));
  {
    ProfScope ps(stream);
    UB_CHECK_CUDA(launch_pdl(kern, grid, dim3(ATT_THREADS), ATT_BWD_SMEM, stream, 1, tmQ, tmD, p, acc));
  }
  UB_CHECK_CUDA(cudaGetLastError());
  {
    ProfScope ps(stream);
    if (di) UB_CHECK_CUDA(launch_pdl(attn_dq_convert_kernel<true>, dim3(a.batch), dim3(256), 0, stream, 1, static_cast<const float*>(acc), a.dqkv, a.cu_seqlens, a.hidden));
    else UB_CHECK_CUDA(launch_pdl(attn_dq_convert_kernel<false>, dim3(a.batch), dim3(256), 0, stream, 1, static_cast<const float*>(acc), a.dqkv, a.cu_seqlens, a.hidden));
    UB_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}
