// C entry point of the wgmma GEMM core: argument checks, tile / cluster selection, TMA
// descriptors.  Device code lives in gemm_impl.cuh (instantiated in gemm_bf16.cu / gemm_f16.cu).
#include "common.h"

#include "gemm_params.h"

namespace ub {
int gemm_dispatch_bf16(int bn, int cluster, int a_major, int b_major, const GemmParams& p,
                       const CUtensorMap& tmA, const CUtensorMap& tmB, int grid, cudaStream_t stream);
int gemm_dispatch_f16(int bn, int cluster, int a_major, int b_major, const GemmParams& p,
                      const CUtensorMap& tmA, const CUtensorMap& tmB, int grid, cudaStream_t stream);
int gemm_group_dispatch_bf16(const void* tm, const GroupedParams& g, int grid, cudaStream_t stream);
int gemm_group_dispatch_f16(const void* tm, const GroupedParams& g, int grid, cudaStream_t stream);

// Every UB200_EPI_* bit the epilogue implements; any other bit is an argument error.
constexpr int EPI_KNOWN = UB200_EPI_BIAS | UB200_EPI_DROPOUT | UB200_EPI_RESIDUAL | UB200_EPI_GELU |
                          UB200_EPI_DGELU | UB200_EPI_ACCUM | UB200_EPI_OUT_F32 | UB200_EPI_COLSUM |
                          UB200_EPI_ATOMIC | UB200_EPI_TANH;

// Pick (N tile, CTAs per tile) minimising the modelled time in microseconds:
//   waves x (k-blocks x per_kb(bn, cluster) + per_tile(bn, cluster)).
// per_kb is the mainloop time of one 128 x bn x 64 step; per_tile is what a wave loses per tile
// beyond its mainloop: the part of the epilogue warpgroup's work that the next mainloop does not
// hide, and the tile switch.  Both grow with the tile width; a 2-CTA cluster fetches each B tile once
// per pair.  Wide tiles amortise the fixed part until wave quantisation bites, which is what makes
// 128-wide tiles win for the N = 3072, K = 768 GEMMs at 27 row tiles (648 tiles = 4.9 waves).
// The constants are a non-negative least-squares fit (relative error) to tools/gemm_roles.py over the
// eight encoder roles, T = 3456 and 3578, every (tile, cluster) below, on an H100 80GB HBM3 at 700 W
// (profiles/h100_c2_gemm_tiles_epilogue_wg.jsonl).  Scored on those explicit-tile timings, the fitted
// choices total 426.1 us over the 16 shapes against 421.2 us for the fastest tile of each shape.  All
// of the gap is at 28 row tiles, in the two N = 3072 roles with the erf epilogues (GELU, dGELU),
// whose tiles are bound by the epilogue warpgroup: there waves x width is the same for 128, 192 and
// 256 (6, 4 and 3 waves), and the model, which knows only (M, N, K), picks 256 (FFN1 fwd 45.5 us
// where 128 gives 42.5; FFN2 dgrad 49.9 us where 192 gives 48.0).  The overlapped form,
// waves x max(mainloop, epilogue) + one epilogue, fitted to the same timings, makes the same choices.
static void pick_config(int M, int N, int K, int sms, int* bn_out, int* cluster_out) {
  const int tiles_m = (M + BM - 1) / BM;
  const int num_kb = (K + BK - 1) / BK;
  const int cand[6][2] = {{256, 2}, {128, 2}, {256, 1}, {192, 1}, {128, 1}, {64, 1}};
  double best = 1e30;
  *bn_out = 128; *cluster_out = 1;
  for (int i = 0; i < 6; ++i) {
    const int bn = cand[i][0], c = cand[i][1];
    if (c == 2 && tiles_m < 2) continue;
    const int units = ((tiles_m + c - 1) / c) * ((N + bn - 1) / bn);
    const int slots = sms / c;
    const int waves = (units + slots - 1) / slots;
    const double per_kb = (c == 1) ? 0.07216 + 0.00234 * bn : 0.00288 * bn;
    const double per_tile = (c == 1) ? 0.12773 + 0.01752 * bn : 0.02067 * bn;
    const double cost = static_cast<double>(waves) * (num_kb * per_kb + per_tile);
    if (cost < best - 1e-9) { best = cost; *bn_out = bn; *cluster_out = c; }
  }
}

// SM count the tile heuristics assume in the deterministic mode (that of an H100 SXM), so that the tile
// shape, and with it every output bit, cannot change with ub200_set_sm_reserve.
constexpr int DET_CONFIG_SMS = 132;

}  // namespace ub

extern "C" int ub200_gemm(const ub200_gemm_args* args, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(args != nullptr, "gemm: args is NULL");
  const ub200_gemm_args& a = *args;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  UB_CHECK_ARG(a.M > 0 && a.N > 0 && a.K > 0, "gemm: M, N, K must be positive (%d, %d, %d)", a.M,
               a.N, a.K);
  UB_CHECK_ARG(a.a != nullptr && a.b != nullptr && a.out != nullptr, "gemm: null operand");
  UB_CHECK_ARG(a.dtype == UB200_F16 || a.dtype == UB200_BF16, "gemm: bad dtype %d", a.dtype);
  UB_CHECK_ARG(a.N % 8 == 0 && a.ldo % 8 == 0, "gemm: N and ldo must be multiples of 8");
  const int epi = a.epilogue;
  UB_CHECK_ARG((epi & ~EPI_KNOWN) == 0, "gemm: unknown epilogue bits 0x%x", epi & ~EPI_KNOWN);
  UB_CHECK_ARG(!(epi & UB200_EPI_BIAS) || a.bias, "gemm: EPI_BIAS without bias");
  UB_CHECK_ARG(!(epi & UB200_EPI_RESIDUAL) || (a.residual && a.ldr % 8 == 0),
               "gemm: EPI_RESIDUAL needs residual with ldr %% 8 == 0");
  UB_CHECK_ARG(!(epi & UB200_EPI_GELU) || a.out2, "gemm: EPI_GELU without out2");
  UB_CHECK_ARG(!(epi & UB200_EPI_DGELU) || (a.aux && a.ldaux % 8 == 0),
               "gemm: EPI_DGELU needs aux with ldaux %% 8 == 0");
  UB_CHECK_ARG(!(epi & UB200_EPI_COLSUM) || (a.colsum && (reinterpret_cast<uintptr_t>(a.colsum) & 15) == 0),
               "gemm: EPI_COLSUM needs a 16-byte aligned colsum (vector atomics)");
  UB_CHECK_ARG(!((epi & UB200_EPI_GELU) && (epi & UB200_EPI_OUT_F32)),
               "gemm: EPI_GELU with fp32 output is not supported");
  UB_CHECK_ARG(a.dropout_p >= 0.f && a.dropout_p < 1.f, "gemm: dropout_p out of range");
  UB_CHECK_ARG(!(epi & UB200_EPI_ATOMIC) || epi == (UB200_EPI_ATOMIC | UB200_EPI_OUT_F32),
               "gemm: EPI_ATOMIC combines with EPI_OUT_F32 only");
  UB_CHECK_ARG(a.k_splits >= -1, "gemm: k_splits must be >= -1");
  UB_CHECK_ARG(a.k_splits == 0 || a.k_splits == 1 || (epi & UB200_EPI_ATOMIC),
               "gemm: k_splits > 1 needs EPI_ATOMIC | EPI_OUT_F32 and a zeroed output");
  UB_CHECK_ARG(a.n_valid >= 0 && a.n_valid <= a.N, "gemm: n_valid must be in [0, N]");
  const int n_valid = a.n_valid ? a.n_valid : a.N;

  if (deterministic() && (epi & (UB200_EPI_COLSUM | UB200_EPI_ATOMIC))) {
    // Fixed-order forms.  Split-K is not used: one CTA sums each output element over all of K and adds
    // it to the (zeroed) output, so the split count can depend on nothing.  The bias gradient is a
    // fixed-order column sum of the 16-bit output, as nn.Linear's bias gradient sums the 16-bit grad.
    UB_CHECK_ARG(!((epi & UB200_EPI_COLSUM) && (epi & UB200_EPI_OUT_F32)),
                 "gemm: EPI_COLSUM needs a 16-bit output in deterministic mode");
    ub200_gemm_args b = a;
    b.epilogue = epi & ~(UB200_EPI_COLSUM | UB200_EPI_ATOMIC);
    if (epi & UB200_EPI_ATOMIC) b.epilogue |= UB200_EPI_ACCUM;
    b.colsum = nullptr;
    b.k_splits = 0;
    const int rc = ub200_gemm(&b, stream_);
    if (rc || !(epi & UB200_EPI_COLSUM)) return rc;
    return launch_colsum_det(a.dtype, a.out, a.colsum, a.M, a.N, a.ldo, stream);
  }

  const int sms = num_sms();
  int bn = 0, cluster = 0;
  // deterministic mode: the tile shape is a function of (M, N, K) only, never of the SM reserve
  pick_config(a.M, a.N, a.K, deterministic() ? DET_CONFIG_SMS : sms, &bn, &cluster);
  if (a.tile_n) {
    bn = a.tile_n;
    if (!a.cluster) cluster = ((bn == 128 || bn == 256) && a.M > BM) ? 2 : 1;
  }
  if (a.cluster) cluster = a.cluster;
  const bool splitk = a.k_splits > 1 || a.k_splits == -1;
  if (splitk) {              // split-K units live in the 1-SM kernel
    cluster = 1;
    if (!a.tile_n) bn = a.N >= 128 ? 128 : 64;
  }
  UB_CHECK_ARG(cluster == 1 || cluster == 2, "gemm: cluster must be 0, 1 or 2 (got %d)", cluster);
  UB_CHECK_ARG(!(cluster == 2 && (bn == 64 || bn == 192)), "gemm: cluster 2 needs tile_n 128 or 256");

  CUtensorMap tmA, tmB;
  int rc;
  if (a.a_major == 0)
    rc = make_tma_2d(&tmA, a.a, a.dtype, a.M, a.K, a.lda, BM, BK);
  else
    rc = make_tma_2d(&tmA, a.a, a.dtype, a.K, a.M, a.lda, BK, 64);
  if (rc) return rc;
  if (a.b_major == 0)  // in 2-CTA clusters each CTA loads (and multicasts) half of the B rows
    rc = make_tma_2d(&tmB, a.b, a.dtype, n_valid, a.K, a.ldb, bn / cluster, BK);
  else
    rc = make_tma_2d(&tmB, a.b, a.dtype, a.K, n_valid, a.ldb, BK, 64);
  if (rc) return rc;

  GemmParams p;
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.epilogue = epi;
  p.bias = a.bias; p.residual = a.residual; p.aux = a.aux;
  p.out = a.out; p.out2 = a.out2; p.colsum = a.colsum;
  p.ldr = a.ldr; p.ldaux = a.ldaux; p.ldo = a.ldo;
  if ((epi & UB200_EPI_DROPOUT) && a.dropout_p > 0.f) {
    const DropoutThreshold d = dropout_threshold(a.dropout_p);
    p.drop_thr16 = d.thr16;
    p.drop_inv_keep = d.inv_keep;
  } else {
    p.epilogue &= ~UB200_EPI_DROPOUT;
    p.drop_thr16 = 0;
    p.drop_inv_keep = 1.f;
  }
  p.seed_lo = static_cast<uint32_t>(a.rng_seed);
  p.seed_hi = static_cast<uint32_t>(a.rng_seed >> 32);
  p.stream_lo = static_cast<uint32_t>(a.rng_stream);
  p.stream_hi = static_cast<uint32_t>(a.rng_stream >> 32);
  p.rng_dev = reinterpret_cast<const unsigned long long*>(a.rng_offset_dev);
  p.tiles_m = (a.M + BM - 1) / BM;
  p.tiles_n = (a.N + bn - 1) / bn;
  const int num_kb = (a.K + BK - 1) / BK;
  p.ksplit = 1;
  p.kb_per_split = num_kb;
  if (splitk) {
    const int tiles = p.tiles_m * p.tiles_n;
    int want = a.k_splits == -1 ? (sms + tiles - 1) / tiles : a.k_splits;
    if (want > num_kb) want = num_kb;
    if (want < 1) want = 1;
    p.kb_per_split = (num_kb + want - 1) / want;
    p.ksplit = (num_kb + p.kb_per_split - 1) / p.kb_per_split;   // every slice has >= 1 k-block
  }
  const int units = ((p.tiles_m + cluster - 1) / cluster) * p.tiles_n * p.ksplit;
  int slots = (a.max_ctas > 0 ? a.max_ctas : sms) / cluster;
  if (slots < 1) slots = 1;
  if (slots > units) slots = units;
  const int grid = slots * cluster;

  if (a.dtype == UB200_BF16)
    return gemm_dispatch_bf16(bn, cluster, a.a_major, a.b_major, p, tmA, tmB, grid, stream);
  return gemm_dispatch_f16(bn, cluster, a.a_major, a.b_major, p, tmA, tmB, grid, stream);
}

extern "C" int ub200_gemm_grouped(const ub200_gemm_args* args, int32_t count, ub200_stream_t stream_) {
  using namespace ub;
  UB_CHECK_ARG(args != nullptr && count >= 1 && count <= GEMM_MAX_GROUP,
               "gemm_grouped: need 1..%d problems", GEMM_MAX_GROUP);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  struct { CUtensorMap a[GEMM_MAX_GROUP]; CUtensorMap b[GEMM_MAX_GROUP]; } tm;
  GroupedParams g{};
  g.nprob = count; g.K = args[0].K; g.epilogue = args[0].epilogue;
  for (int i = 0; i < count; ++i) {
    const ub200_gemm_args& a = args[i];
    UB_CHECK_ARG(a.a && a.b && a.out, "gemm_grouped[%d]: null operand", i);
    UB_CHECK_ARG(a.a_major == 1 && a.b_major == 1, "gemm_grouped[%d]: operands must be MN-major (wgrad form)", i);
    UB_CHECK_ARG(a.K == g.K && a.dtype == args[0].dtype && a.epilogue == g.epilogue,
                 "gemm_grouped[%d]: K / dtype / epilogue must match problem 0", i);
    UB_CHECK_ARG(a.M > 0 && a.N > 0 && a.K > 0 && a.N % 8 == 0 && a.ldo % 8 == 0,
                 "gemm_grouped[%d]: bad shape", i);
  }
  // N tile shared by the group: fewest (rounds over the SMs) x (cost per k-block of a 128 x bn tile,
  // an unmeasured heuristic, not part of pick_config's fit: wider tiles cost less per column).
  const int sms = num_sms();
  int bn = args[0].tile_n;
  if (bn == 0) {
    double best = 1e30;
    const int cand[3] = {128, 192, 256};
    for (int c = 0; c < 3; ++c) {
      int t = 0;
      for (int i = 0; i < count; ++i) t += ((args[i].M + BM - 1) / BM) * ((args[i].N + cand[c] - 1) / cand[c]);
      const int cs = deterministic() ? DET_CONFIG_SMS : sms;   // tile shape independent of the SM reserve
      const double cost = static_cast<double>((t + cs - 1) / cs) * (421.0 + 1.27 * cand[c]);
      if (cost < best - 1e-9) { best = cost; bn = cand[c]; }
    }
  }
  UB_CHECK_ARG(bn == 128 || bn == 192 || bn == 256, "gemm_grouped: tile_n must be 0, 128, 192 or 256 (got %d)", bn);
  g.bn = bn;
  int tiles = 0;
  for (int i = 0; i < count; ++i) {
    const ub200_gemm_args& a = args[i];
    int rc = make_tma_2d(&tm.a[i], a.a, a.dtype, a.K, a.M, a.lda, BK, 64);
    if (rc) return rc;
    rc = make_tma_2d(&tm.b[i], a.b, a.dtype, a.K, a.N, a.ldb, BK, 64);
    if (rc) return rc;
    g.M[i] = a.M; g.N[i] = a.N; g.out[i] = a.out; g.ldo[i] = a.ldo;
    g.tiles_n[i] = (a.N + bn - 1) / bn;
    g.tile_start[i] = tiles;
    tiles += ((a.M + BM - 1) / BM) * g.tiles_n[i];
  }
  for (int i = count; i <= GEMM_MAX_GROUP; ++i) g.tile_start[i] = tiles;
  for (int i = count; i < GEMM_MAX_GROUP; ++i) { tm.a[i] = tm.a[0]; tm.b[i] = tm.b[0]; }
  int grid = sms;
  if (grid > tiles) grid = tiles;
  if (args[0].dtype == UB200_BF16) return gemm_group_dispatch_bf16(&tm, g, grid, stream);
  return gemm_group_dispatch_f16(&tm, g, grid, stream);
}
