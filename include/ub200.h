/*
 * ub200.h — C ABI of the H100-native UNITER encoder hot path (libub200.so).
 *
 * The reference (ChenRocks/UNITER) is pure Python: its "FFI" for this path is the set of
 * torch / apex / horovod library calls made by model/layer.py and model/model.py.  Each entry
 * point below replaces one group of those call sites (cited as <file>:<lines> under the
 * reference root).  Rules of the boundary (SURVEY.md §8b-B2):
 *   - plain C: raw device pointers, explicit sizes / leading dimensions, POD structs;
 *   - the CALLER owns all memory (outputs, saved tensors, workspaces are pre-allocated);
 *   - no allocation, no host synchronisation, no exceptions across the ABI;
 *   - every launch goes onto the cudaStream_t passed in (never the legacy default stream);
 *   - return 0 on success, a negative UB200_E* code otherwise; ub200_last_error_string()
 *     gives the message for the calling thread.
 *
 * Data layout: activations are PACKED — row t of a [T, H] matrix is the t-th valid token of
 * the batch (sequence b occupies rows cu_seqlens[b] .. cu_seqlens[b+1]); there is no padding.
 * 16-bit storage type is selected by `dtype` (UB200_F16 / UB200_BF16); accumulation, softmax
 * and LayerNorm statistics are fp32.
 */
#ifndef UB200_H_
#define UB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* ub200_stream_t; /* == cudaStream_t */

enum { UB200_F16 = 0, UB200_BF16 = 1 };

enum {
  UB200_OK = 0,
  UB200_EINVAL = -1,      /* bad argument (null pointer, misaligned, negative size) */
  UB200_EUNSUPPORTED = -2, /* shape outside what the kernels implement */
  UB200_ECUDA = -3,       /* CUDA runtime / driver error, see last_error_string */
};

/* library identity ------------------------------------------------------------------------ */
int ub200_version(void);                      /* MAJOR*10000 + MINOR*100 + PATCH */
const char* ub200_last_error_string(void);    /* thread-local, never NULL */
int ub200_device_check(void);                 /* 0 iff the current device is sm_90 (H100) */

/* launch accounting / profiling (used by bench.py: "gpu_launches" and the roofline pass).
 * Tags: 0 untagged (gather / convert), 1 qkv GEMM, 2 attention fwd, 3 attn-out GEMM, 4 LN1 fwd,
 * 5 FFN1 GEMM, 6 FFN2 GEMM, 7 LN2 fwd, 8 LN2 bwd, 9 FFN2 dgrad, 10 FFN2 wgrad, 11 FFN1 dgrad,
 * 12 FFN1 wgrad, 13 LN1 bwd, 14 attn-out dgrad, 15 attn-out wgrad, 16 attention bwd,
 * 17 dbias column sum, 18 QKV dgrad, 19 QKV wgrad, 20 gradient add. */
unsigned long long ub200_launch_count(void);  /* kernels launched by this library so far */
/* Persistent kernels of this library size their grids to the SM count.  While a collective (NCCL)
 * runs concurrently on another stream its CTAs occupy SMs; a persistent CTA that cannot be placed
 * starts a whole round late.  `n` SMs are left free by every later launch (0 restores the full
 * device); returns the previous value.  Used by uniter_b200.distributed.GradientReducer while the
 * chunked all-reduce overlaps the backward pass (replaces utils/distributed.py:16-43). */
int ub200_set_sm_reserve(int n);
/* Deterministic mode (on != 0; returns the previous value).  Read at launch time, like the SM reserve,
 * so a captured CUDA graph keeps the mode it was captured under.  With the mode on, the reductions
 * below use no floating-point atomics and no summation order that depends on the grid (so neither the
 * SM reserve nor appended all-zero padding rows change their bits): a whole training step with
 * sequences of at most 128 tokens is bit-reproducible in this mode.  The Python package sets it from
 * torch.use_deterministic_algorithms (see DESIGN.md section 3b).  The forms it selects:
 *   column sums (ub200_colsum, UB200_EPI_COLSUM, the attention's dbias, the LayerNorm backward's
 *     dgamma / dbeta / dbias, ub200_embed_bwd_colsums): one CTA owns 8 columns, thread t sums rows
 *     t, t + 256, ... in ascending order, the 256 partials meet in a fixed tree;
 *   UB200_EPI_COLSUM sums the 16-bit output after the GEMM instead of the fp32 values in its epilogue;
 *   k_splits / UB200_EPI_ATOMIC: no split-K, each element is summed over all of K by one CTA;
 *   ub200_layernorm_bwd: always the split form, so stats_ws is REQUIRED (rows x 2 floats), for the
 *     row_kind / dropout_on_dy cases too;
 *   ub200_embed_bwd_scatter: each table row is owned by the first packed row with that id, which sums
 *     all its rows in ascending order in fp32 and adds to the table once (hidden <= 1024);
 *   ub200_grad_sumsq is an error: use ub200_grad_sumsq_ws (one partial per ub200_adam_chunk() block,
 *     summed in block order);
 *   ub200_attn_bwd: max_seqlen <= 128 only (UB200_EUNSUPPORTED otherwise);
 *   the GEMM tile shape is chosen for 132 SMs whatever the reserve.
 * Nothing changes with the mode off. */
int ub200_set_deterministic(int on);
int ub200_deterministic(void);            /* the current value */
int ub200_profile_enable(int on);
int ub200_profile_collect(float* ms_per_tag, int* launches_per_tag, int ntags);

/* ------------------------------------------------------------------------------------------
 * GEMM core:  D[M,N] = epilogue( sum_k A[m,k] * B[n,k] )      (wgmma + TMA, fp32 accumulate)
 *
 * Replaces every nn.Linear on the path and its autograd mirror:
 *   forward  model/layer.py:76-78 (query/key/value), :112 (attention.output.dense),
 *            :140 (intermediate.dense) + :31-37 (erf GELU), :153 (output.dense);
 *   backward torch autograd of the same nn.Linear modules (dgrad: B is MN-major = the weight
 *            read un-transposed; wgrad: A and B MN-major = activations read un-transposed).
 *
 * Operand storage:
 *   a_major == 0 : A is [M, K] row-major (K contiguous),  lda = row pitch in elements
 *   a_major == 1 : A is [K, M] row-major (M contiguous),  lda = row pitch in elements
 *   b_major == 0 : B is [N, K] row-major (K contiguous)   -- an nn.Linear weight as stored
 *   b_major == 1 : B is [K, N] row-major (N contiguous)
 * Epilogue, applied in this order to v = acc[m,n]:
 *   UB200_EPI_BIAS      v += bias[n]
 *   UB200_EPI_DROPOUT   v = keep(m,n) ? v / (1-p) : 0          (Philox, regenerated in bwd)
 *   UB200_EPI_RESIDUAL  v += residual[m,n]
 *   UB200_EPI_GELU      out2[m,n] = v ; v = gelu_erf(v)         (model/layer.py:31-37)
 *   UB200_EPI_TANH      v = tanh(v)                              (BertPooler, model/layer.py:184)
 *   UB200_EPI_DGELU     v *= gelu_erf'(aux[m,n])
 *   UB200_EPI_ACCUM     v += out[m,n]   (previous contents, e.g. gradient accumulation)
 *   UB200_EPI_OUT_F32   out is fp32 instead of the 16-bit dtype
 *   UB200_EPI_COLSUM    colsum[n] += sum_m v  (fp32 atomics; bias gradients)
 *   UB200_EPI_ATOMIC    out[m,n] += v with fp32 atomics (requires OUT_F32 and a pre-zeroed out);
 *                       the only epilogue allowed with k_splits > 1 (split-K partial sums)
 * Any other bit of `epilogue` is UB200_EINVAL.
 * ------------------------------------------------------------------------------------------ */
enum {
  UB200_EPI_BIAS = 1,
  UB200_EPI_DROPOUT = 2,
  UB200_EPI_RESIDUAL = 4,
  UB200_EPI_GELU = 8,
  UB200_EPI_DGELU = 16,
  UB200_EPI_ACCUM = 32,
  UB200_EPI_OUT_F32 = 64,
  UB200_EPI_COLSUM = 128,
  UB200_EPI_ATOMIC = 256,
  UB200_EPI_TANH = 512,
};

typedef struct {
  const void* a;
  const void* b;
  int64_t lda, ldb;
  int32_t a_major, b_major;
  int32_t M, N, K;
  int32_t dtype;
  int32_t epilogue;        /* OR of UB200_EPI_* */
  const void* bias;        /* [N] 16-bit */
  const void* residual;    /* [M, N] 16-bit, pitch ldr */
  const void* aux;         /* [M, N] 16-bit, pitch ldaux (pre-activation for DGELU) */
  void* out;               /* [M, N], pitch ldo */
  void* out2;              /* [M, N] 16-bit, pitch ldo (pre-activation, GELU only) */
  float* colsum;           /* [N] fp32, accumulated with (16-byte vector) atomics: 16-byte aligned */
  int64_t ldr, ldaux, ldo;
  float dropout_p;         /* 0 <= p < 1 */
  uint64_t rng_seed;       /* Philox key */
  uint64_t rng_stream;     /* distinguishes dropout sites / layers / steps */
  int32_t tile_n;          /* 0 = heuristic, else force 64 / 128 / 192 / 256 */
  int32_t max_ctas;        /* 0 = one CTA per SM */
  int32_t cluster;         /* 0 = heuristic, 1 = single CTAs, 2 = 2-CTA clusters sharing B by
                              TMA multicast */
  int32_t k_splits;        /* 0 / 1 = none; n > 1: K is cut into <= n slices that run as independent
                              work units (few output tiles, long K: the MLM decoder's dgrad) and meet
                              through UB200_EPI_ATOMIC; -1 = as many as fill the SMs */
  int32_t n_valid;         /* 0 = N; else B only holds n_valid of the N output features (rows if
                              b_major == 0, columns if b_major == 1): the rest contribute acc = 0.
                              Lets N be padded to a multiple of 8 over an unpadded weight (the tied
                              decoder [28996, H] of model/layer.py:206-222) */
  const uint64_t* rng_offset_dev; /* optional DEVICE counter: the dropout stream used is
                              rng_stream + (*rng_offset_dev << 20).  Lets a CUDA graph replay the same
                              launch with fresh masks (the host bumps the counter, not the arguments) */
} ub200_gemm_args;

int ub200_gemm(const ub200_gemm_args* args, ub200_stream_t stream);

/* Up to 4 weight-gradient GEMMs (a_major = b_major = 1, same K / dtype, epilogue 0 or
 * UB200_EPI_ACCUM) as ONE persistent launch: the autograd mirror of the four nn.Linear modules of
 * a BertLayer (model/layer.py:76-78,112,140,153), issued once at the end of the layer's backward. */
int ub200_gemm_grouped(const ub200_gemm_args* args, int32_t count, ub200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused variable-length multi-head self-attention (head_dim 64), forward and backward.
 *
 * Replaces model/layer.py:80-100 (transpose_for_scores, QK^T, /sqrt(d), +mask, softmax, dropout,
 * PV, permute+contiguous) and its autograd mirror.  `qkv` is the packed [T, 3H] output of the
 * fused query|key|value projection; sequence b owns rows cu_seqlens[b] .. cu_seqlens[b+1] and
 * only attends inside that range (the reference's additive -10000 key mask underflows to a
 * probability of exactly 0, so omitting masked keys is exact).  ctx is [T, H]; lse is
 * [num_heads, T] fp32 (log-sum-exp of the scaled scores, saved for backward).
 * Backward reads qkv, ctx, lse, dctx and writes dqkv [T, 3H]; sequences longer than 128 tokens
 * need `workspace` of ub200_attn_bwd_workspace_bytes() bytes.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const void* qkv;            /* [T, 3H] 16-bit */
  void* ctx;                  /* [T, H] 16-bit (output of fwd, input of bwd) */
  float* lse;                 /* [num_heads, T] */
  const int32_t* cu_seqlens;  /* [batch + 1], device */
  int32_t batch, total_tokens, max_seqlen, hidden, num_heads, dtype;
  float dropout_p;            /* attention_probs_dropout_prob when training, else 0 */
  uint64_t rng_seed, rng_stream;
  const void* dctx;           /* bwd: [T, H] */
  void* dqkv;                 /* bwd: [T, 3H] */
  void* workspace;            /* bwd: fp32 dQ accumulator or NULL */
  float* dbias;               /* bwd, optional: [3H] fp32, += column sums of dqkv = gradient of the
                                 stacked query|key|value biases (fused; saves a pass over dqkv) */
  const uint64_t* rng_offset_dev; /* optional device counter added to rng_stream (see ub200_gemm_args) */
} ub200_attn_args;

int ub200_attn_fwd(const ub200_attn_args* args, ub200_stream_t stream);
int ub200_attn_bwd(const ub200_attn_args* args, ub200_stream_t stream);
int64_t ub200_attn_bwd_workspace_bytes(int32_t total_tokens, int32_t hidden, int32_t max_seqlen);

/* ------------------------------------------------------------------------------------------
 * Row-wise kernels (HBM-bound, 16-byte vector accesses, fp32 statistics).
 *
 * ub200_layernorm_fwd / _bwd replace apex FusedLayerNorm(eps=1e-12) at model/layer.py:108,114,
 * 149,155 and model/model.py:228,243,254-259,270 (biased variance, eps inside the sqrt).  The
 * backward also produces, in the same pass, dgamma / dbeta, the dropout-masked copy of dx that
 * feeds the preceding Linear's dgrad / wgrad (dropout at model/layer.py:113,154 regenerated from
 * the Philox stream used by the forward GEMM epilogue) and that Linear's bias gradient.
 * ub200_gather_rows is the bit-exact row mover behind pack / unpack and the gather_index
 * compaction of model/model.py:330-333:  dst[r] = index[r] >= 0 ? src[index[r]] : 0.
 *
 * Rows are up to 2048 columns wide (hidden % 8 == 0).  act = UB200_LN_ACT_RELU normalises relu(x)
 * instead of x: y = LN(relu(pre)), the Linear(H, 2H) -> ReLU -> LayerNorm(2H) of the VCR head
 * (model/vcr.py:27-32), with `pre` the Linear's 16-bit output.  Its backward takes pre as `x` and
 * writes dpre = dx o (pre > 0) to dx_drop (required; dropout_p must be 0), with dbias = the column sums
 * of dpre.  ReLU rows and rows wider than 1024 take the split form (stats_ws required) on plain rows.
 * ------------------------------------------------------------------------------------------ */
#define UB200_LN_ACT_NONE 0
#define UB200_LN_ACT_RELU 1

int ub200_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, int32_t rows,
                        int32_t hidden, int32_t dtype, ub200_stream_t stream);
int ub200_layernorm_fwd_act(const void* x, const void* gamma, const void* beta, void* y, int32_t rows,
                            int32_t hidden, int32_t dtype, int32_t act, ub200_stream_t stream);

typedef struct {
  const void* dy;     /* [rows, hidden] */
  const void* x;      /* [rows, hidden] input of the forward LayerNorm (pre-LN residual sum) */
  const void* gamma;  /* [hidden] */
  void* dx;           /* [rows, hidden] */
  void* dx_drop;      /* [rows, hidden] dx * mask / keep, required iff dropout_p > 0 */
  float* dgamma;      /* [hidden] fp32, accumulated; dgamma / dbeta / dbias 16-byte aligned */
  float* dbeta;       /* [hidden] fp32, accumulated */
  float* dbias;       /* [hidden] fp32 column sum of the Linear-branch gradient, or NULL */
  int32_t rows, hidden, dtype;
  float dropout_p;
  uint64_t rng_seed, rng_stream;
  const int32_t* row_kind;  /* optional [rows]: only rows with row_kind[r] == kind are processed
                               (the embedding front-end has different LayerNorms per row kind) */
  int32_t kind;
  int32_t dropout_on_dy;    /* bit 0: y = dropout(LN(x)) (embeddings): mask dy instead of emitting dx_drop;
                               bit 1: with row_kind, rows of the OTHER kind get dx = 0 (else untouched) */
  const uint64_t* rng_offset_dev; /* optional device counter added to rng_stream (see ub200_gemm_args) */
  float* stats_ws;          /* optional scratch, rows x 2 floats: selects the split form (a row kernel that
                               carries nothing between rows + a column-reduction kernel) for the plain
                               case (no row_kind, dropout on the Linear branch); NULL = one fused kernel */
  int32_t act;              /* UB200_LN_ACT_NONE, or UB200_LN_ACT_RELU: x is pre of y = LN(relu(pre)) */
} ub200_ln_bwd_args;
int ub200_layernorm_bwd(const ub200_ln_bwd_args* args, ub200_stream_t stream);

int ub200_gather_rows(const void* src, void* dst, const int32_t* index, int32_t rows,
                      int32_t row_bytes, ub200_stream_t stream);
int ub200_colsum(const void* x, float* out, int32_t rows, int32_t cols, int64_t ld, int32_t dtype,
                 ub200_stream_t stream);
int ub200_cvt_from_f32(const float* src, void* dst, int64_t n, int32_t accumulate, int32_t dtype,
                       ub200_stream_t stream);
/* nseg segments of n elements: dst[s*dst_stride + j] (+)= 16-bit(src[s*src_stride + j]) — the small
 * (bias / LayerNorm) gradients of several encoder layers finalised in one launch. */
int ub200_cvt_from_f32_strided(const float* src, void* dst, int64_t n, int64_t nseg,
                               int64_t src_stride, int64_t dst_stride, int32_t accumulate,
                               int32_t dtype, ub200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Whole encoder stack: NL x BertLayer forward / backward in ONE call each, so that the host
 * enqueues ~7 (fwd) / ~13 (bwd) kernels per layer from C++ without returning to Python.
 *
 * Replaces UniterEncoder.forward (model/model.py:282-292) = NL x BertLayer.forward
 * (model/layer.py:166-170): BertSelfAttention (:75-101), BertSelfOutput (:111-115),
 * BertIntermediate (:139-142), BertOutput (:152-156), and the autograd graph behind them.
 *
 * Per layer (x = previous layer output, packed [T, H]):
 *   qkv = x Wqkv^T + bqkv                              GEMM, bias epilogue
 *   ctx = attention(qkv)                               fused varlen attention
 *   s1  = dropout(ctx Wo^T + bo) + x                   GEMM, bias + dropout + residual epilogue
 *   a   = LayerNorm(s1)
 *   pre = a W1^T + b1 ; f = gelu_erf(pre)              GEMM, bias + GELU epilogue (both kept)
 *   s2  = dropout(f W2^T + b2) + a                     GEMM, bias + dropout + residual epilogue
 *   out = LayerNorm(s2)
 * Weights stay where the nn.Parameters live; query/key/value must be stacked contiguously
 * ([3H, H] and [3H]) — the Python module guarantees that by making the three parameters views
 * of one buffer.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const void *wqkv, *bqkv;    /* [3H, H], [3H]   attention.self.{query,key,value} stacked */
  const void *wo, *bo;        /* [H, H], [H]     attention.output.dense */
  const void *ln1_g, *ln1_b;  /* [H]             attention.output.LayerNorm */
  const void *w1, *b1;        /* [I, H], [I]     intermediate.dense */
  const void *w2, *b2;        /* [H, I], [H]     output.dense */
  const void *ln2_g, *ln2_b;  /* [H]             output.LayerNorm */
} ub200_layer_weights;

typedef struct {
  void *dwqkv, *dwo, *dw1, *dw2; /* 16-bit, same shapes as the weights */
  float* small;                  /* fp32, ub200_encoder_small_grad_count() entries, accumulated:
                                    dbqkv[3H] dbo[H] dln1_g[H] dln1_b[H] db1[I] db2[H] dln2_g[H] dln2_b[H] */
} ub200_layer_grads;

typedef struct {
  int32_t hidden, intermediate, num_heads, num_layers, dtype;
  int32_t batch, total_tokens, max_seqlen;
  const int32_t* cu_seqlens;     /* device, [batch + 1] */
  float hidden_dropout_p;        /* 0 when not training */
  float attn_dropout_p;
  uint64_t rng_seed, rng_offset; /* rng_offset must differ between forward calls */
  int32_t layer_offset;          /* index of layers[0] in the whole stack (dropout streams are keyed
                                    by the global layer index, so a backward may be issued in chunks) */
  const uint64_t* rng_offset_dev; /* optional DEVICE counter added to rng_offset at run time: a captured
                                    CUDA graph of the step draws new dropout masks on every replay */
} ub200_encoder_desc;

/* bytes of saved activations per layer (fwd writes, bwd reads) and of backward scratch */
int64_t ub200_encoder_act_bytes_per_layer(const ub200_encoder_desc* d);
int64_t ub200_encoder_bwd_scratch_bytes(const ub200_encoder_desc* d);
int64_t ub200_encoder_small_grad_count(int32_t hidden, int32_t intermediate);

/* x_in [T, H]; layer_out[l] -> [T, H] output of layer l (caller-allocated, NL pointers);
 * act: NL * act_bytes_per_layer when save_for_backward, else one layer's worth (reused). */
int ub200_encoder_fwd(const ub200_encoder_desc* d, const ub200_layer_weights* layers,
                      const void* x_in, void* const* layer_out, void* act,
                      int32_t save_for_backward, ub200_stream_t stream);

/* d_layer_out[l]: gradient wrt layer_out[l] or NULL (at least the last must be given);
 * dx_in [T, H] receives the gradient wrt x_in; accumulate_wgrad != 0 adds into dW*. */
int ub200_encoder_bwd(const ub200_encoder_desc* d, const ub200_layer_weights* layers,
                      const ub200_layer_grads* grads, const void* x_in,
                      void* const* layer_out, const void* act, const void* const* d_layer_out,
                      void* dx_in, void* scratch, int32_t accumulate_wgrad,
                      ub200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Embedding front-end, computed straight into packed rows (model/model.py:217-334).
 *
 * ub200_embed_prep: per packed row t (= position pack_idx[t] = b*L + j of the attention mask)
 *   src = gather_index[b, j] (joint mode) or j; text row iff src < Lt.  Emits int32 arrays
 *   kind (0 text / 1 image), word_id, pos_id, type_id, img_src (= b*Li + region or -1),
 *   mask_flag (img_masks).  Pure integer logic: bit-exact by construction.
 * ub200_embed_gather_cast: out[t] = 16-bit(img_feat[img_src[t]] (+ mask_row if mask_flag[t])),
 *   zeros for text rows  ->  A operand [T, D] of the img_linear GEMM (ub200_gemm, bias epilogue).
 * ub200_embed_rows_fwd: text  x = dropout(LN_txt(word + pos + type))             (:232-245)
 *                       image x = dropout(LN_out(LN_img(G) + LN_pos(box W^T + b) + type)) (:261-272)
 *   u (pre-final-LN sum) and ppre (pos_linear output) are saved for the backward, which is
 *   ub200_layernorm_bwd with row_kind masks + wgrad GEMMs + table scatter.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const int32_t* pack_idx;     /* [T] */
  const int64_t* gather_index; /* [B, L] (joint) */
  const int64_t* input_ids;    /* [B, Lt] */
  const int64_t* position_ids; /* [pos_rows, Lt], pos_rows = 1 (broadcast) or B */
  const int64_t* txt_type_ids; /* [B, Lt] or NULL (0) */
  const int64_t* img_type_ids; /* [B, Li] or NULL (1) */
  const uint8_t* img_masks;    /* [B, Li] bool/uint8 or NULL */
  int32_t T, L, Lt, Li, pos_rows, mode;   /* mode: 0 joint, 1 text only, 2 image only */
  int32_t *kind, *word_id, *pos_id, *type_id, *img_src, *mask_flag;   /* outputs, [T] each */
} ub200_embed_prep_args;
int ub200_embed_prep(const ub200_embed_prep_args* args, ub200_stream_t stream);

int ub200_embed_gather_cast(const void* img_feat, int32_t feat_is_f32, const int32_t* img_src,
                            const int32_t* mask_flag, const void* mask_row, void* out, int32_t T,
                            int32_t D, int32_t dtype, ub200_stream_t stream);

typedef struct {
  const int32_t *kind, *word_id, *pos_id, *type_id, *img_src;          /* from ub200_embed_prep */
  const void *word_emb, *pos_emb, *type_emb;                           /* embedding tables, 16-bit */
  const void *ln_txt_g, *ln_txt_b;                                     /* embeddings.LayerNorm */
  const void* img_linear_out;                                          /* [T, H] 16-bit */
  const float* pos_feat;                                               /* [B*Li, 7] fp32 */
  const void *w_pos, *b_pos;                                           /* pos_linear [H,7], [H] */
  const void *ln_img_g, *ln_img_b, *ln_pos_g, *ln_pos_b, *ln_out_g, *ln_out_b;
  void *x, *u, *ppre;                                                  /* [T, H] 16-bit outputs */
  int32_t T, hidden, dtype;
  float dropout_p;
  uint64_t rng_seed, rng_stream;
  const uint64_t* rng_offset_dev; /* optional device counter added to rng_stream (see ub200_gemm_args) */
} ub200_embed_rows_args;
int ub200_embed_rows_fwd(const ub200_embed_rows_args* args, ub200_stream_t stream);


/* Backward of the embedding front-end's table lookups (autograd mirror of model/model.py:235-237,
 * :258, :316-317), after ub200_layernorm_bwd produced du (gradient wrt the pre-LayerNorm sums) and
 * dP (gradient wrt the pos_linear output, zero on text rows):
 *   ub200_embed_bwd_scatter   text rows: d_word[word_id[t]] += du[t] (16-bit packed atomics into the
 *                             pre-zeroed [V, H] gradient), d_pos[pos_id[t]] += du[t] (fp32)
 *   ub200_embed_bwd_colsums   mode 0: d_type[ty, :] += sum_{t: type_id[t]==ty} x[t, :]     ([Ty, H] fp32)
 *                             mode 1: d_wpos[h, k] += sum_{image rows t} x[t, h] * box[t, k] ([H, 7] fp32,
 *                                     box = pos_feat[img_src[t]] rounded to the 16-bit dtype)
 * fp32 outputs are accumulated (caller zeroes them). */
int ub200_embed_bwd_scatter(const void* du, const int32_t* kind, const int32_t* word_id,
                            const int32_t* pos_id, void* d_word, float* d_pos, int32_t T,
                            int32_t hidden, int32_t dtype, ub200_stream_t stream);
typedef struct {
  const void* x;             /* [T, hidden] 16-bit: du (mode 0) or dP (mode 1) */
  const int32_t* type_id;    /* mode 0 */
  const int32_t* kind;       /* mode 1 */
  const int32_t* img_src;    /* mode 1 */
  const float* pos_feat;     /* mode 1: [B*Li, 7] fp32 */
  float* out;                /* mode 0: [type_vocab, hidden]; mode 1: [hidden, 7] */
  int32_t T, hidden, mode, type_vocab, dtype;
} ub200_embed_colsum_args;
int ub200_embed_bwd_colsums(const ub200_embed_colsum_args* args, ub200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Callers either side of the encoder (SURVEY.md §8f-1, -2).
 *
 * MLM head (model/layer.py:188-222 BertPredictionHeadTransform + tied decoder, model/pretrain.py:
 * 107-127): dense+GELU, LayerNorm and the decoder run on ub200_gemm / ub200_layernorm_*; these
 * are the pieces in between.  `logits` is [rows, ld] 16-bit with ld >= vocab rounded up to 8.
 *   ub200_ce_fwd   loss[r] = logsumexp(logits[r, :vocab]) - logits[r, target[r]], lse[r] saved
 *                  (F.cross_entropy(..., reduction='none'); targets outside [0, vocab) -> 0)
 *   ub200_ce_bwd   dlogits[r, c] = (softmax - onehot) * dloss[r] for c < vocab, 0 for
 *                  vocab <= c < ncols; dlogits may alias logits
 *   ub200_dgelu_mul  out = dy * gelu_erf'(pre)   (n elements, n % 8 == 0)
 *   ub200_dtanh_mul  out = dy * (1 - y^2), y = tanh(pre) as saved by the forward: backward of
 *                    BertPooler (model/layer.py:179-185), whose forward is ub200_gemm with UB200_EPI_TANH
 * ------------------------------------------------------------------------------------------ */
int ub200_ce_fwd(const void* logits, int64_t ld, const int64_t* targets, float* loss, float* lse,
                 int32_t rows, int32_t vocab, int32_t dtype, ub200_stream_t stream);
int ub200_ce_bwd(const void* logits, void* dlogits, int64_t ld, const int64_t* targets,
                 const float* lse, const float* dloss, int32_t rows, int32_t vocab, int32_t ncols,
                 int32_t dtype, ub200_stream_t stream);
int ub200_dgelu_mul(const void* dy, const void* pre, void* out, int64_t n, int32_t dtype,
                    ub200_stream_t stream);
int ub200_dtanh_mul(const void* dy, const void* y, void* out, int64_t n, int32_t dtype,
                    ub200_stream_t stream);

/* Referring-expression head (model/re.py:48-100): one Linear(H, 1) score per image region and the
 * per-sample loss over a sample's regions.  `rows` is a [R, H] 16-bit matrix of region rows (H % 8 ==
 * 0, 16-byte aligned); sample b owns rows seg_start[b] .. seg_start[b] + seg_len[b] - 1 (int32 device
 * tables).  Segments are disjoint and ascending; rows outside every segment are padding.  One CTA per
 * sample.  Per sample b and region k < max_regions:
 *   score[b, k] = round16(rows[seg_start[b] + k] . weight + bias)     (fp32 accumulation)
 *   score[b, k] = round16(-1e4) where k >= seg_len[b] or obj_masks[b, k] != 0   (masked_fill)
 * and, for targets t = targets[b] in [0, seg_len[b]) (others: loss 0, no gradient):
 *   UB200_RE_CLS   loss[b] = logsumexp(score[b, :]) - score[b, t] in fp32; lse[b] saved
 *   UB200_RE_RANK  loss[b] = max(margin + sigmoid(score[b, n]) - sigmoid(score[b, t]), 0), where
 *                  n = neg_plan[b] if >= 0 (an easy negative drawn by the caller), and for
 *                  neg_plan[b] == -1 the highest-scoring unmasked region != t (ties: lowest index);
 *                  the chosen n is saved in neg_ix[b]
 * The backward writes dscore = dloss * (softmax - onehot) (cls) or -+ sigmoid'(s) * dloss at t / n
 * where the hinge is >= 0 (rank), 0 at masked positions;  d_rows[r] = round16(dscore * weight) for the
 * rows of every segment and 0 for padding rows;  dweight[H] = sum dscore * rows and dbias[0] = sum
 * dscore in fp32, written (not accumulated).  The two weight sums are per-sample partials (workspace)
 * added in sample order by a second launch: no float atomics, the same bits in every mode. */
enum { UB200_RE_SCORES = 0, UB200_RE_CLS = 1, UB200_RE_RANK = 2 };
typedef struct {
  const void* rows;          /* [R, H] */
  const void* weight;        /* [H] */
  const void* bias;          /* [1] or NULL */
  const int32_t* seg_start;  /* [batch] */
  const int32_t* seg_len;    /* [batch] */
  const uint8_t* obj_masks;  /* [batch, max_regions], non-zero = masked (uint8 or bool) */
  const int64_t* targets;    /* [batch] (cls / rank) */
  const int64_t* neg_plan;   /* [batch] (rank) */
  void* scores;              /* [batch, max_regions] 16-bit */
  float* loss;               /* [batch] (cls / rank) */
  float* lse;                /* [batch] (cls) */
  int32_t* neg_ix;           /* [batch] (rank) */
  const float* dloss;        /* [batch] (backward) */
  void* d_rows;              /* [R, H] (backward) */
  float* dweight;            /* [H] (backward) */
  float* dbias;              /* [1] (backward) */
  void* workspace;           /* >= ub200_region_score_workspace_bytes (backward) */
  int64_t workspace_bytes;
  int32_t R, hidden, batch, max_regions, mode, dtype;
  float margin;
} ub200_region_score_args;
int64_t ub200_region_score_workspace_bytes(int32_t batch, int32_t hidden);
int ub200_region_score_fwd(const ub200_region_score_args* args, ub200_stream_t stream);
int ub200_region_score_bwd(const ub200_region_score_args* args, ub200_stream_t stream);

/* Word-region alignment (model/ot.py, model/pretrain.py:166-193): the IPOT optimal-transport distance
 * between the text rows and the region rows of each image-text pair, read straight from the packed
 * [total_rows, H] 16-bit encoder output.  Pair b owns rows cu_seqlens[b] .. cu_seqlens[b+1] - 1: its
 * m = txt_len[b] text rows x_i first, then its n regions y_j (int32 device tables).  One CTA per pair.
 *   x^ = x / max(|x|, 1e-5), y^ likewise (fp32 row norms);  C[i, j] = 1 - x^_i . y^_j, the dot products
 *   on tensor cores (mma.sync m16n8k16, 16-bit inputs, fp32 accumulation);
 *   IPOT with beta 0.5, 50 iterations, k = 1 (model/ot.py:36-67): sigma = 1/m, T = 1, A = exp(-C^T/beta);
 *   each iteration Q = A * T, delta = 1/(n Q sigma), sigma = 1/(m delta^T Q), T = delta * Q * sigma;
 *   dist[b] = round16(sum_ij C[i, j] T[j, i]), stored as fp32.
 * C, A and T of a pair stay in shared memory for all 50 iterations; the forward saves T and the row
 * norms in the workspace.  The backward treats T as a constant: with g = d_dist[b], dC = g T^T, then
 * dx^ = -dC y^, dy^ = -dC^T x^ and the F.normalize backward give d_packed for every row of every pair;
 * rows from cu_seqlens[batch] to total_rows - 1 get 0.  Fixed summation orders, no float atomics.
 * Supported: hidden a multiple of 16 up to 1024, and max_m * max_n <= UB200_WRA_MAX_MN (11 x 1024:
 * three fp32 [n, m] matrices and four fp32 vectors fit the 227 KB of shared memory of one H100 CTA even
 * at m + n = m n + 1), UB200_EUNSUPPORTED otherwise.  max_m < 1 or max_n < 1 is UB200_EINVAL.  A pair
 * outside 1 <= m <= max_m, 1 <= n <= max_n (device values the host does not see) gets dist NaN and a
 * zero gradient. */
#define UB200_WRA_MAX_MN 11264
typedef struct {
  const void* packed;          /* [total_rows, H] */
  const int32_t* cu_seqlens;   /* [batch + 1] */
  const int32_t* txt_len;      /* [batch] */
  float* dist;                 /* [batch] (forward) */
  const float* d_dist;         /* [batch] (backward) */
  void* d_packed;              /* [total_rows, H] (backward) */
  void* workspace;             /* >= ub200_wra_workspace_bytes: written by the forward, read by the backward */
  int64_t workspace_bytes;
  int32_t total_rows, hidden, batch, max_m, max_n, dtype;
} ub200_wra_args;
int64_t ub200_wra_workspace_bytes(int32_t batch, int32_t max_m, int32_t max_n);
int ub200_wra_fwd(const ub200_wra_args* args, ub200_stream_t stream);
int ub200_wra_bwd(const ub200_wra_args* args, ub200_stream_t stream);

/* Multi-tensor AdamW on fp32 master weights: replaces optim/adamw.py:43-103 (+ the apex O2
 * master-gradient copy, unscale and master->model copy around it, train_vqa.py:152,190-227) and
 * torch.nn.utils.clip_grad_norm_ (train_vqa.py:223-226).  One segment per parameter tensor;
 * `segs` and `blk_start` (int32 [nseg + 1], prefix sums of ceil(n / ub200_adam_chunk())) live in
 * DEVICE memory, nblocks = blk_start[nseg].  Per element, with g = grad * inv_scale * clip:
 *   m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; p -= step_size * m / (sqrt(v) + eps) ;
 *   p -= lr_wd * p  (lr * weight_decay, AFTER the Adam update) ; model = round16(p)
 * step_size = lr * sqrt(1 - b2^t) / (1 - b1^t) (or lr without bias correction) is computed by
 * the caller per segment.  clip = min(1, max_norm / (sqrt(sumsq) * inv_scale + 1e-6)) is read
 * from the device scalar written by ub200_grad_sumsq (no host synchronisation). */
typedef struct {
  const void* grad;       /* [n] gradient in grad_dtype */
  float* master;          /* [n] fp32 master weights */
  float* exp_avg;         /* [n] fp32 */
  float* exp_avg_sq;      /* [n] fp32 */
  void* model;            /* [n] model weights in model_dtype, or NULL */
  int64_t n;
  float step_size;
  float lr_wd;
  int32_t grad_dtype;     /* UB200_F16 / UB200_BF16 / UB200_F32 */
  int32_t model_dtype;
  /* device-state mode (ub200_adam_state given to ub200_adamw_step): */
  float weight_decay;     /* lr_wd = lr * weight_decay with lr = lr_dev[group] */
  int32_t group;          /* index into lr_dev */
  int32_t step_offset;    /* this tensor's step count = state->step - step_offset (a parameter that got
                             its first gradient later than the others) */
  int32_t flags;          /* bit 0: bias-corrected step size (optim/adamw.py:82-86) */
} ub200_adam_segment;

/* Device-resident optimizer state: lets a whole training step (loss scaling included) run without
 * the host ever reading a gradient — apex amp's dynamic loss scaler (train_vqa.py:152,190-192) skips
 * the step when a gradient overflowed; here ub200_adam_prep decides that ON THE DEVICE from the sum of
 * squares: found_inf = !isfinite(sumsq); a finite step increments `step`, an overflowed one increments
 * `skipped` and ub200_adamw_step leaves masters, moments and model weights untouched. */
typedef struct {
  int32_t step;       /* number of optimizer steps actually applied */
  int32_t found_inf;  /* 1 iff the last ub200_adam_prep saw a non-finite gradient norm */
  int32_t skipped;    /* number of skipped (overflowed) steps */
  int32_t _pad;
} ub200_adam_state;
int ub200_adam_prep(const float* sumsq, ub200_adam_state* state_dev, ub200_stream_t stream);  /* ordinary launch, no PDL */
enum { UB200_F32 = 2 };
int32_t ub200_adam_chunk(void);
int ub200_grad_sumsq(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev, int32_t nseg,
                     int32_t nblocks, float* out, ub200_stream_t stream);
/* ub200_grad_sumsq with caller-owned scratch of ub200_grad_sumsq_workspace_bytes(nblocks) bytes (4-byte
 * aligned), which the deterministic mode needs (a smaller one is UB200_EINVAL); with the mode off the
 * workspace is not touched. */
int64_t ub200_grad_sumsq_workspace_bytes(int32_t nblocks);
int ub200_grad_sumsq_ws(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev, int32_t nseg,
                        int32_t nblocks, float* out, void* workspace, int64_t workspace_bytes,
                        ub200_stream_t stream);
/* state_dev / lr_dev NULL: legacy mode (host-computed step_size / lr_wd per segment, no skipping).
 * Otherwise: skip when state->found_inf; lr = lr_dev[seg.group]; bias correction from state->step. */
int ub200_adamw_step(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev, int32_t nseg,
                     int32_t nblocks, float beta1, float beta2, float eps, float inv_scale,
                     float max_norm, const float* sumsq, const ub200_adam_state* state_dev,
                     const float* lr_dev, ub200_stream_t stream);

/* Device-resident dynamic loss scaling (apex amp's LossScaler in dynamic mode, train_vqa.py:152,189-199;
 * pre-training keeps one scaler per task, pretrain.py:230-233,298-301): a table of entries, one per
 * loss id, in DEVICE memory at a fixed address.  The caller multiplies its loss by `scale` on the
 * device before the backward; ub200_adam_prep_scaled (instead of ub200_adam_prep, after
 * ub200_grad_sumsq) sets found_inf / step / skipped exactly as ub200_adam_prep does, records
 * inv_scale = 1 / scale (what this step's gradients carry), then updates entry `loss_id` only:
 *   overflow:  scale = max(scale / 2, min_scale) (plain scale / 2 when min_scale <= 0), unskipped = 0
 *   otherwise: unskipped += 1; when unskipped == window: scale = min(scale * 2, max_scale), unskipped = 0
 * ub200_adamw_step_scaled is ub200_adamw_step in device-state mode with the unscale factor read from
 * the entry's inv_scale (gradient multiplier and clip norm alike).  No host read anywhere: a whole
 * fp16 step, loss scale included, replays from one CUDA graph.  apex defaults: scale 2^16,
 * window 2000, max_scale 2^24, no floor.  loss_id must index the caller's table.  The prep kernel is
 * an ordinary launch with full dependencies on ub200_grad_sumsq before it and ub200_adamw_step_scaled
 * after it (not a programmatic dependent), so the overflow check holds inside captured graphs. */
typedef struct {
  float scale;        /* current loss scale */
  int32_t unskipped;  /* clean steps since the scale last changed */
  float inv_scale;    /* 1 / scale of the step the last ub200_adam_prep_scaled ran for */
  int32_t window;     /* clean steps before the scale doubles (apex scale_seq_len) */
  float max_scale;    /* growth cap */
  float min_scale;    /* floor on overflow; <= 0: none */
  int32_t _pad[2];
} ub200_loss_scaler;
int ub200_adam_prep_scaled(const float* sumsq, ub200_adam_state* state_dev, ub200_loss_scaler* scalers_dev,
                           int32_t loss_id, ub200_stream_t stream);
int ub200_adamw_step_scaled(const ub200_adam_segment* segs_dev, const int32_t* blk_start_dev, int32_t nseg,
                            int32_t nblocks, float beta1, float beta2, float eps, float max_norm,
                            const float* sumsq, const ub200_adam_state* state_dev, const float* lr_dev,
                            const ub200_loss_scaler* scalers_dev, int32_t loss_id, ub200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Gradient exchange over NVLink peer memory — replaces utils/distributed.py:16-43
 * (all_reduce_and_rescale_tensors: flatten -> hvd.allreduce_ = mean over ranks -> unflatten; call
 * sites train_vqa.py:193-199, pretrain.py:302-308).  One call averages one slice of the flat gradient
 * arena over the ranks, two-shot: push my copy of sub-slice q to rank q's staging buffer, flag barrier,
 * reduce sub-slice `rank` in fp32 (rank order 0..world-1, so every rank ends up with bit-identical
 * values), write it into every rank's arena, flag barrier.  Everything the call enqueues is an
 * ordinary node of the caller's stream / CUDA graph (no host synchronisation, no NCCL).  `max_ctas`
 * selects who moves the bytes:
 *   < 0  the copy engines (cudaMemcpyAsync nodes); 32-thread kernels run the flag barriers and one kernel
 *        reduces out of local HBM — the form to overlap with compute (it uses no SM for the transfers);
 *   = 0  a push kernel + a reduce kernel of short-lived CTAs (256 threads) sized by the work;
 *   > 0  ONE persistent kernel of that many CTAs (256 threads x <= 64 registers, no shared memory:
 *        a CTA fits next to a persistent GEMM CTA), posted remote stores.
 *
 * Memory (caller-owned, one set per rank, mapped into every process with the ipc calls below):
 *   buf[q]   rank q's arena base (16-bit elements); the slice is [offset, offset + count)
 *   stage[q] rank q's staging buffer, >= ub200_peer_stage_bytes(count, world) bytes
 *   flags[q] rank q's signal block, ub200_peer_flags_bytes() bytes, zero-initialised ONCE (epochs
 *            are monotonic); word 19 is a sticky error word: non-zero after a wait expired
 *            (value = (call number << 4) | phase) — the data of that and later calls is invalid.
 * Every rank must issue the same sequence of calls (same offset / count), one at a time per rank. */
#define UB200_MAX_PEERS 8
typedef struct {
  void* buf[UB200_MAX_PEERS];
  void* stage[UB200_MAX_PEERS];
  uint32_t* flags[UB200_MAX_PEERS];
  int32_t rank, world;
  int64_t offset, count;     /* elements; both multiples of 8 (16 bytes) */
  int64_t stage_bytes;       /* size of each staging buffer */
  int32_t dtype;             /* UB200_F16 / UB200_BF16 */
  int32_t max_ctas;          /* form of the exchange, see above (< 0: copy engines) */
  float scale;               /* result = scale * sum over ranks; 1/world = Horovod's average */
  int32_t timeout_ms;        /* bound of every flag wait (0: 20 s) */
} ub200_peer_allreduce_args;
int64_t ub200_peer_flags_bytes(void);
int64_t ub200_peer_stage_bytes(int64_t count, int32_t world);
int ub200_peer_allreduce(const ub200_peer_allreduce_args* args, ub200_stream_t stream);
/* cudaIpc plumbing for device memory owned by the caller (e.g. a torch caching-allocator block):
 * export gives the 64-byte handle of the ALLOCATION containing dev_ptr and dev_ptr's byte offset in
 * it; open maps that allocation into this process (peer access is enabled lazily) and returns its
 * base; an allocation may be opened once per process. */
int ub200_peer_ipc_export(const void* dev_ptr, void* handle64, int64_t* offset_bytes);
int ub200_peer_ipc_open(const void* handle64, void** mapped_base);
int ub200_peer_ipc_close(void* mapped_base);

#ifdef __cplusplus
}
#endif
#endif /* UB200_H_ */
