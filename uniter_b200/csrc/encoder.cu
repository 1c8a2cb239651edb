// Encoder-stack orchestration: enqueues the per-layer kernel sequence of NL BertLayers
// (forward and backward) from C++ so that one C-ABI call covers the whole stack.
// Reference: UniterEncoder.forward model/model.py:282-292, BertLayer model/layer.py:159-170.
#include "common.h"

namespace ub {

static inline int64_t align256(int64_t v) { return (v + 255) & ~static_cast<int64_t>(255); }

// Saved activations of one layer (16-bit unless noted), in workspace order.
struct ActLayout {
  int64_t qkv, ctx, s1, a, pre, f, s2, lse, total;
  ActLayout(int64_t T, int64_t H, int64_t I, int64_t heads) {
    int64_t o = 0;
    qkv = o; o += align256(T * 3 * H * 2);
    ctx = o; o += align256(T * H * 2);
    s1 = o;  o += align256(T * H * 2);
    a = o;   o += align256(T * H * 2);
    pre = o; o += align256(T * I * 2);
    f = o;   o += align256(T * I * 2);
    s2 = o;  o += align256(T * H * 2);
    lse = o; o += align256(heads * T * 4);
    total = o;
  }
};

struct BwdScratch {
  int64_t bufA, bufB, bufC, bufD, bufE, g0, g1, dpre, dqkv, attn_ws, ln_stats, total;
  BwdScratch(int64_t T, int64_t H, int64_t I, int64_t attn_ws_bytes) {
    int64_t o = 0;
    bufA = o; o += align256(T * H * 2);   // ds2
    bufB = o; o += align256(T * H * 2);   // dy2 (dropout-masked ds2)
    bufC = o; o += align256(T * H * 2);   // da, then dctx
    bufD = o; o += align256(T * H * 2);   // ds1
    bufE = o; o += align256(T * H * 2);   // dy1 (dropout-masked ds1)
    g0 = o;   o += align256(T * H * 2);
    g1 = o;   o += align256(T * H * 2);
    dpre = o; o += align256(T * I * 2);
    dqkv = o; o += align256(T * 3 * H * 2);
    attn_ws = o; o += align256(attn_ws_bytes);
    ln_stats = o; o += align256(T * 2 * 4);   // (mean, rstd) per row for the split LayerNorm backward
    total = o;
  }
};

// offsets inside ub200_layer_grads.small
struct SmallLayout {
  int64_t dbqkv, dbo, dg1, db1ln, db1, db2, dg2, db2ln, total;
  SmallLayout(int64_t H, int64_t I) {
    int64_t o = 0;
    dbqkv = o; o += 3 * H;
    dbo = o;   o += H;
    dg1 = o;   o += H;
    db1ln = o; o += H;
    db1 = o;   o += I;
    db2 = o;   o += H;
    dg2 = o;   o += H;
    db2ln = o; o += H;
    total = o;
  }
};

static int check_desc(const ub200_encoder_desc* d, const char* who) {
  if (!d) return set_error(UB200_EINVAL, "%s: desc is NULL", who);
  if (d->hidden <= 0 || d->hidden % 64 != 0 || d->num_heads * 64 != d->hidden)
    return set_error(UB200_EUNSUPPORTED, "%s: hidden must equal 64 * num_heads (hidden=%d heads=%d)",
                     who, d->hidden, d->num_heads);
  if (d->hidden > 1024)
    return set_error(UB200_EUNSUPPORTED, "%s: hidden %d > 1024 not supported by the LayerNorm kernels",
                     who, d->hidden);
  if (d->intermediate <= 0 || d->intermediate % 8 != 0)
    return set_error(UB200_EINVAL, "%s: intermediate must be a positive multiple of 8", who);
  if (d->num_layers <= 0 || d->batch <= 0 || d->total_tokens <= 0 || !d->cu_seqlens)
    return set_error(UB200_EINVAL, "%s: empty problem", who);
  if (d->max_seqlen <= 0 || d->max_seqlen > 512)
    return set_error(UB200_EUNSUPPORTED, "%s: max_seqlen %d outside (0, 512]", who, d->max_seqlen);
  if (d->dtype != UB200_F16 && d->dtype != UB200_BF16)
    return set_error(UB200_EINVAL, "%s: bad dtype", who);
  return 0;
}

static inline uint64_t rng_stream_of(const ub200_encoder_desc* d, int layer, int site) {
  return (d->rng_offset << 20) | (static_cast<uint64_t>(layer + d->layer_offset) << 4) |
         static_cast<uint64_t>(site);
}
enum { SITE_ATTN_PROBS = 1, SITE_ATTN_OUT = 2, SITE_FFN_OUT = 3 };

static ub200_gemm_args gemm_base(const ub200_encoder_desc* d) {
  ub200_gemm_args g{};
  g.dtype = d->dtype;
  g.rng_seed = d->rng_seed;
  g.rng_offset_dev = d->rng_offset_dev;
  return g;
}

}  // namespace ub

#define UB_TRY(expr)            \
  do {                          \
    int _rc = (expr);           \
    if (_rc != 0) return _rc;   \
  } while (0)

extern "C" int64_t ub200_encoder_act_bytes_per_layer(const ub200_encoder_desc* d) {
  if (!d) return 0;
  return ub::ActLayout(d->total_tokens, d->hidden, d->intermediate, d->num_heads).total;
}

extern "C" int64_t ub200_encoder_bwd_scratch_bytes(const ub200_encoder_desc* d) {
  if (!d) return 0;
  const int64_t ws = ub200_attn_bwd_workspace_bytes(d->total_tokens, d->hidden, d->max_seqlen);
  return ub::BwdScratch(d->total_tokens, d->hidden, d->intermediate, ws).total;
}

extern "C" int64_t ub200_encoder_small_grad_count(int32_t hidden, int32_t intermediate) {
  return ub::SmallLayout(hidden, intermediate).total;
}

extern "C" int ub200_encoder_fwd(const ub200_encoder_desc* d, const ub200_layer_weights* layers,
                                 const void* x_in, void* const* layer_out, void* act_,
                                 int32_t save_for_backward, ub200_stream_t stream) {
  using namespace ub;
  UB_TRY(check_desc(d, "encoder_fwd"));
  UB_CHECK_ARG(layers && x_in && layer_out && act_, "encoder_fwd: null pointer");
  const int T = d->total_tokens, H = d->hidden, I = d->intermediate;
  const ActLayout L(T, H, I, d->num_heads);
  uint8_t* act = reinterpret_cast<uint8_t*>(act_);

  const void* x = x_in;
  for (int l = 0; l < d->num_layers; ++l) {
    const ub200_layer_weights& w = layers[l];
    uint8_t* A = act + (save_for_backward ? static_cast<int64_t>(l) * L.total : 0);
    UB_CHECK_ARG(layer_out[l], "encoder_fwd: layer_out[%d] is NULL", l);

    // qkv = x Wqkv^T + bqkv                                   model/layer.py:76-78
    ub200_gemm_args g = gemm_base(d);
    g.a = x; g.lda = H; g.b = w.wqkv; g.ldb = H; g.M = T; g.N = 3 * H; g.K = H;
    g.epilogue = UB200_EPI_BIAS; g.bias = w.bqkv; g.out = A + L.qkv; g.ldo = 3 * H;
    {
      ProfTag _t(1);
      UB_TRY(ub200_gemm(&g, stream));
    }

    // ctx = softmax(q k^T / 8 [keys of the same sequence]) v   model/layer.py:80-100
    ub200_attn_args at{};
    at.qkv = A + L.qkv; at.ctx = A + L.ctx; at.lse = reinterpret_cast<float*>(A + L.lse);
    at.cu_seqlens = d->cu_seqlens; at.batch = d->batch; at.total_tokens = T;
    at.max_seqlen = d->max_seqlen; at.hidden = H; at.num_heads = d->num_heads; at.dtype = d->dtype;
    at.dropout_p = d->attn_dropout_p; at.rng_seed = d->rng_seed;
    at.rng_stream = rng_stream_of(d, l, SITE_ATTN_PROBS);
    at.rng_offset_dev = d->rng_offset_dev;
    {
      ProfTag _t(2);
      UB_TRY(ub200_attn_fwd(&at, stream));
    }

    // s1 = dropout(ctx Wo^T + bo) + x ; a = LayerNorm(s1)       model/layer.py:112-114
    g = gemm_base(d);
    g.a = A + L.ctx; g.lda = H; g.b = w.wo; g.ldb = H; g.M = T; g.N = H; g.K = H;
    g.epilogue = UB200_EPI_BIAS | UB200_EPI_RESIDUAL | (d->hidden_dropout_p > 0 ? UB200_EPI_DROPOUT : 0);
    g.bias = w.bo; g.residual = x; g.ldr = H; g.out = A + L.s1; g.ldo = H;
    g.dropout_p = d->hidden_dropout_p; g.rng_stream = rng_stream_of(d, l, SITE_ATTN_OUT);
    {
      ProfTag _t(3);
      UB_TRY(ub200_gemm(&g, stream));
    }
    {
      ProfTag _t(4);
      UB_TRY(ub200_layernorm_fwd(A + L.s1, w.ln1_g, w.ln1_b, A + L.a, T, H, d->dtype, stream));
    }

    // pre = a W1^T + b1 ; f = gelu(pre)                        model/layer.py:140-141, :31-37
    g = gemm_base(d);
    g.a = A + L.a; g.lda = H; g.b = w.w1; g.ldb = H; g.M = T; g.N = I; g.K = H;
    g.epilogue = UB200_EPI_BIAS | UB200_EPI_GELU;
    g.bias = w.b1; g.out = A + L.f; g.out2 = A + L.pre; g.ldo = I;
    {
      ProfTag _t(5);
      UB_TRY(ub200_gemm(&g, stream));
    }

    // s2 = dropout(f W2^T + b2) + a ; out = LayerNorm(s2)      model/layer.py:153-155
    g = gemm_base(d);
    g.a = A + L.f; g.lda = I; g.b = w.w2; g.ldb = I; g.M = T; g.N = H; g.K = I;
    g.epilogue = UB200_EPI_BIAS | UB200_EPI_RESIDUAL | (d->hidden_dropout_p > 0 ? UB200_EPI_DROPOUT : 0);
    g.bias = w.b2; g.residual = A + L.a; g.ldr = H; g.out = A + L.s2; g.ldo = H;
    g.dropout_p = d->hidden_dropout_p; g.rng_stream = rng_stream_of(d, l, SITE_FFN_OUT);
    {
      ProfTag _t(6);
      UB_TRY(ub200_gemm(&g, stream));
    }
    {
      ProfTag _t(7);
      UB_TRY(ub200_layernorm_fwd(A + L.s2, w.ln2_g, w.ln2_b, layer_out[l], T, H, d->dtype, stream));
    }
    x = layer_out[l];
  }
  return 0;
}

namespace ub {
int launch_add16(int dtype, void* dst, const void* a, const void* b, long long n, cudaStream_t stream);
}

extern "C" int ub200_encoder_bwd(const ub200_encoder_desc* d, const ub200_layer_weights* layers,
                                 const ub200_layer_grads* grads, const void* x_in,
                                 void* const* layer_out, const void* act_,
                                 const void* const* d_layer_out, void* dx_in, void* scratch_,
                                 int32_t accumulate_wgrad, ub200_stream_t stream) {
  using namespace ub;
  UB_TRY(check_desc(d, "encoder_bwd"));
  UB_CHECK_ARG(layers && grads && x_in && layer_out && act_ && d_layer_out && dx_in && scratch_,
               "encoder_bwd: null pointer");
  const int NL = d->num_layers;
  UB_CHECK_ARG(d_layer_out[NL - 1], "encoder_bwd: gradient of the last layer output is required");
  const int T = d->total_tokens, H = d->hidden, I = d->intermediate;
  const ActLayout L(T, H, I, d->num_heads);
  const SmallLayout SG(H, I);
  const int64_t attn_ws = ub200_attn_bwd_workspace_bytes(T, H, d->max_seqlen);
  const BwdScratch S(T, H, I, attn_ws);
  const uint8_t* act = reinterpret_cast<const uint8_t*>(act_);
  uint8_t* sc = reinterpret_cast<uint8_t*>(scratch_);
  cudaStream_t cs = reinterpret_cast<cudaStream_t>(stream);
  const bool drop = d->hidden_dropout_p > 0.f;
  const int acc = accumulate_wgrad ? UB200_EPI_ACCUM : 0;
  // the deterministic mode's LayerNorm backward (row kernel + fixed-order column kernel) needs stats_ws
  float* ln_ws = deterministic() ? reinterpret_cast<float*>(sc + S.ln_stats) : nullptr;

  const void* dcur = d_layer_out[NL - 1];
  int pp = 0;  // ping-pong for the running gradient
  for (int l = NL - 1; l >= 0; --l) {
    const ub200_layer_weights& w = layers[l];
    const ub200_layer_grads& gr = grads[l];
    UB_CHECK_ARG(gr.dwqkv && gr.dwo && gr.dw1 && gr.dw2 && gr.small, "encoder_bwd: grads[%d] has NULLs", l);
    const uint8_t* A = act + static_cast<int64_t>(l) * L.total;
    const void* x = (l == 0) ? x_in : layer_out[l - 1];
    void* dnext = (l == 0) ? dx_in : (sc + (pp ? S.g1 : S.g0));
    pp ^= 1;

    // ---- out = LN(s2): ds2 (bufA), dropout-masked copy (bufB), dgamma/dbeta, db2
    ub200_ln_bwd_args ln{};
    ln.dy = dcur; ln.x = A + L.s2; ln.gamma = w.ln2_g; ln.dx = sc + S.bufA;
    ln.dx_drop = drop ? sc + S.bufB : nullptr;
    ln.dgamma = gr.small + SG.dg2; ln.dbeta = gr.small + SG.db2ln; ln.dbias = gr.small + SG.db2;
    ln.rows = T; ln.hidden = H; ln.dtype = d->dtype; ln.dropout_p = d->hidden_dropout_p;
    ln.rng_seed = d->rng_seed; ln.rng_stream = rng_stream_of(d, l, SITE_FFN_OUT);
    ln.rng_offset_dev = d->rng_offset_dev; ln.stats_ws = ln_ws;
    {
      ProfTag _t(8);
      UB_TRY(ub200_layernorm_bwd(&ln, stream));
    }
    const void* dy2 = drop ? sc + S.bufB : sc + S.bufA;

    // ---- dPre = (dY2 W2) o gelu'(pre) ; db1 = colsum(dPre)
    ub200_gemm_args g = gemm_base(d);
    g.a = dy2; g.lda = H; g.b = w.w2; g.ldb = I; g.b_major = 1; g.M = T; g.N = I; g.K = H;
    g.epilogue = UB200_EPI_DGELU | UB200_EPI_COLSUM; g.aux = A + L.pre; g.ldaux = I;
    g.colsum = gr.small + SG.db1; g.out = sc + S.dpre; g.ldo = I;
    {
      ProfTag _t(9);
      UB_TRY(ub200_gemm(&g, stream));
    }
    // ---- da = dPre W1 + ds2   (bufC)
    g = gemm_base(d);
    g.a = sc + S.dpre; g.lda = I; g.b = w.w1; g.ldb = H; g.b_major = 1; g.M = T; g.N = H; g.K = I;
    g.epilogue = UB200_EPI_RESIDUAL; g.residual = sc + S.bufA; g.ldr = H; g.out = sc + S.bufC; g.ldo = H;
    {
      ProfTag _t(11);
      UB_TRY(ub200_gemm(&g, stream));
    }

    // ---- a = LN(s1): ds1 (bufD), masked copy (bufE), dgamma/dbeta, dbo
    ln = ub200_ln_bwd_args{};
    ln.dy = sc + S.bufC; ln.x = A + L.s1; ln.gamma = w.ln1_g; ln.dx = sc + S.bufD;
    ln.dx_drop = drop ? sc + S.bufE : nullptr;
    ln.dgamma = gr.small + SG.dg1; ln.dbeta = gr.small + SG.db1ln; ln.dbias = gr.small + SG.dbo;
    ln.rows = T; ln.hidden = H; ln.dtype = d->dtype; ln.dropout_p = d->hidden_dropout_p;
    ln.rng_seed = d->rng_seed; ln.rng_stream = rng_stream_of(d, l, SITE_ATTN_OUT);
    ln.rng_offset_dev = d->rng_offset_dev; ln.stats_ws = ln_ws;
    {
      ProfTag _t(13);
      UB_TRY(ub200_layernorm_bwd(&ln, stream));
    }
    const void* dy1 = drop ? sc + S.bufE : sc + S.bufD;

    // ---- dctx = dY1 Wo   (bufC; da is dead after the LayerNorm backward)
    g = gemm_base(d);
    g.a = dy1; g.lda = H; g.b = w.wo; g.ldb = H; g.b_major = 1; g.M = T; g.N = H; g.K = H;
    g.out = sc + S.bufC; g.ldo = H;
    {
      ProfTag _t(14);
      UB_TRY(ub200_gemm(&g, stream));
    }

    // ---- attention backward: dqkv
    ub200_attn_args at{};
    at.qkv = A + L.qkv; at.ctx = const_cast<uint8_t*>(A + L.ctx);
    at.lse = reinterpret_cast<float*>(const_cast<uint8_t*>(A + L.lse));
    at.cu_seqlens = d->cu_seqlens; at.batch = d->batch; at.total_tokens = T;
    at.max_seqlen = d->max_seqlen; at.hidden = H; at.num_heads = d->num_heads; at.dtype = d->dtype;
    at.dropout_p = d->attn_dropout_p; at.rng_seed = d->rng_seed;
    at.rng_stream = rng_stream_of(d, l, SITE_ATTN_PROBS);
    at.rng_offset_dev = d->rng_offset_dev;
    at.dctx = sc + S.bufC; at.dqkv = sc + S.dqkv; at.workspace = attn_ws ? sc + S.attn_ws : nullptr;
    at.dbias = gr.small + SG.dbqkv;   // dbqkv = colsum(dqkv), fused into the attention backward
    {
      ProfTag _t(16);
      UB_TRY(ub200_attn_bwd(&at, stream));
    }
    // ---- dx = dqkv Wqkv + ds1  -> gradient wrt the layer input
    g = gemm_base(d);
    g.a = sc + S.dqkv; g.lda = 3 * H; g.b = w.wqkv; g.ldb = H; g.b_major = 1; g.M = T; g.N = H; g.K = 3 * H;
    g.epilogue = UB200_EPI_RESIDUAL; g.residual = sc + S.bufD; g.ldr = H; g.out = dnext; g.ldo = H;
    {
      ProfTag _t(18);
      UB_TRY(ub200_gemm(&g, stream));
    }

    // ---- the four weight gradients of the layer as ONE grouped launch (all contract over T):
    //      dW2[H,I] = dY2^T f ; dW1[I,H] = dPre^T a ; dWo[H,H] = dY1^T ctx ; dWqkv[3H,H] = dQKV^T x
    {
      ub200_gemm_args wg[4];
      for (int i = 0; i < 4; ++i) {
        wg[i] = gemm_base(d);
        wg[i].a_major = 1; wg[i].b_major = 1; wg[i].K = T; wg[i].epilogue = acc;
      }
      wg[0].a = dy2; wg[0].lda = H; wg[0].b = A + L.f; wg[0].ldb = I;
      wg[0].M = H; wg[0].N = I; wg[0].out = gr.dw2; wg[0].ldo = I;
      wg[1].a = sc + S.dpre; wg[1].lda = I; wg[1].b = A + L.a; wg[1].ldb = H;
      wg[1].M = I; wg[1].N = H; wg[1].out = gr.dw1; wg[1].ldo = H;
      wg[2].a = sc + S.dqkv; wg[2].lda = 3 * H; wg[2].b = x; wg[2].ldb = H;
      wg[2].M = 3 * H; wg[2].N = H; wg[2].out = gr.dwqkv; wg[2].ldo = H;
      wg[3].a = dy1; wg[3].lda = H; wg[3].b = A + L.ctx; wg[3].ldb = H;
      wg[3].M = H; wg[3].N = H; wg[3].out = gr.dwo; wg[3].ldo = H;
      ProfTag _t(10);
      UB_TRY(ub200_gemm_grouped(wg, 4, stream));
    }

    // gradient flowing into the previous layer's output (+ its external gradient, if any)
    if (l > 0 && d_layer_out[l - 1]) {
      {
      ProfTag _t(20);
      UB_TRY(launch_add16(d->dtype, dnext, dnext, d_layer_out[l - 1], static_cast<long long>(T) * H, cs));
    }
    }
    dcur = dnext;
  }
  return 0;
}
