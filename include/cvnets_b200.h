/*
 * cvnets_b200.h -- C ABI of libcvnets_b200.so: the sm_90a kernels behind the apple/ml-cvnets vision-backbone hot path.
 *
 * The reference (apple/ml-cvnets) is pure Python and has NO native operator / FFI boundary (SURVEY.md 8b); its hot
 * path bottoms out in torch.nn.functional calls.  This header is therefore the boundary a maintainer would bind with
 * ctypes/cffi/pybind from the reference's layers (INTEGRATION.md shows the stub).  Each entry point names the
 * reference call site(s) it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *  - plain pointers + sizes only (no torch types); every pointer is a DEVICE pointer unless stated otherwise;
 *  - activations are bf16, channels-last: a feature map [B,H,W,C] is the row-major matrix [M=B*H*W, C];
 *  - parameters / statistics are fp32, batch statistics accumulators are fp64 (atomically accumulated, caller zeroes);
 *  - every function enqueues work on `stream` and returns immediately: 0 on success, non-zero on error
 *    (cvb_last_error() gives the message).  No host sync, no global state: CUDA-graph capturable, DDP safe.
 *  - leading dimensions are in ELEMENTS and must be multiples of 8 (16-byte vector access).
 */
#ifndef CVNETS_B200_H_
#define CVNETS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* cvb_stream_t; /* cudaStream_t */

#if defined(__GNUC__)
#define CVB_API __attribute__((visibility("default")))
#else
#define CVB_API
#endif

#define CVB_ABI_VERSION 12

/* operand "load modes": the normalisation / activation of the PRODUCER layer is applied while the CONSUMER loads it
 * (training-mode BatchNorm cannot be fused into its own conv: SURVEY.md section 7 "hard parts"). */
enum {
  CVB_A_RAW = 0,      /* x                                                                                   */
  CVB_A_AFF = 1,      /* p0[c]*x + p1[c]                 BatchNorm apply (batch_norm.py:14-49)               */
  CVB_A_AFF_SILU = 2, /* silu(p0[c]*x + p1[c])           BatchNorm + Swish (activation/swish.py:13-20)       */
  CVB_A_SILU = 3,     /* silu(x)                                                                             */
  CVB_A_GN = 4,       /* (x-mean[b])*rstd[b]*p0[c]+p1[c] GroupNorm(1,C) = layer_norm_2d (layer_norm.py:75-108) */
  CVB_A_BNB = 5       /* p0[c]*x + p1[c]*x2 + p2[c]      BatchNorm backward dy from (dz, y)  (SURVEY App. A1) */
};

/* epilogue modes of cvb_pw_gemm */
enum {
  CVB_E_STORE = 0,    /* out = acc + bias (+R)                                                               */
  CVB_E_SILU = 1,     /* out = silu(acc + bias) (+R)                                                         */
  CVB_E_SILU_BWD = 2, /* out = acc * silu'(e_p0[n]*Y + e_p1[n]);   col_sum += out, col_sq += out*Y           */
  CVB_E_GN_BWD = 3,   /* xh=(Y-mean[b])*rstd[b]; col_sum += acc, col_sq += acc*xh; out = acc*e_p0[n];
                         samp_sum += out, samp_sq += out*xh   (GroupNorm backward, phase 1)                   */
  CVB_E_LIN_BWD = 4   /* out = acc;   col_sum += out, col_sq += out*Y    (BatchNorm-backward statistics of a producer whose
                         BatchNorm has NO activation: the consumer of a lazily normalised module output)      */
};

CVB_API const char* cvb_last_error(void);
CVB_API int cvb_abi_version(void);
/* host-side query: number of SMs / compute capability of the current device */
CVB_API int cvb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------------------------------------
 * Pointwise (1x1) convolution / linear layer as a GEMM:  C[M,N] = epi( load(A)[M,K] * W[N,K]^T + bias )
 * Replaces F.conv2d(k=1) in ConvLayer2d (cvnets/layers/conv_layer.py:200-226) for InvertedResidual exp_1x1/red_1x1
 * (cvnets/modules/mobilenetv2.py:182-219), MobileViTBlockv2 local_rep[1]/conv_proj (cvnets/modules/mobilevit_block.py
 * :380-412), LinearSelfAttention qkv_proj/out_proj (cvnets/layers/linear_attention.py:51-70), the LinearAttnFFN convs
 * (cvnets/modules/transformer.py:206-226), F.linear of the classifier (cvnets/layers/linear_layer.py:90), and -- with
 * pre-transposed weights -- their input-gradient GEMMs.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct {
  int M, N, K;
  const void* A; int lda;   /* bf16 [M, lda] */
  const void* A2; int lda2; /* bf16 [M, lda2], CVB_A_BNB only */
  int a_mode;
  const float* a_p0; const float* a_p1; const float* a_p2; /* per-K vectors, see load modes */
  const float* row_mean; const float* row_rstd;            /* per-sample [M/rows_per_sample] (CVB_A_GN, CVB_E_GN_BWD) */
  int rows_per_sample;
  const void* W; int ldw;   /* bf16 [N, ldw], K contiguous */
  const float* bias;        /* fp32 [N] or NULL */
  int e_mode;
  const void* Y; int ldy;   /* bf16 [M, ldy] auxiliary tensor of the epilogue (SILU_BWD / GN_BWD) */
  const float* e_p0; const float* e_p1; /* per-N vectors (NULL => 1 / 0) */
  const void* R; int ldr;   /* bf16 [M, ldr] residual added to the output, or NULL */
  void* C; int ldc; int c_fp32; /* output bf16 (or fp32 if c_fp32) [M, ldc] */
  double* col_sum; double* col_sq;   /* fp64 [N] accumulators or NULL (BatchNorm statistics of the stored output) */
  double* samp_sum; double* samp_sq; /* fp64 [M/rows_per_sample] or NULL (GroupNorm statistics of the stored output) */
  double* gn_ws;            /* CVB_E_GN_BWD only, optional: ZEROED fp64 workspace [2][M/rows_per_sample][N].  When given (and
                               rows_per_sample % 64 == 0) the epilogue runs on the wgmma kernel: it accumulates the per-(sample, channel)
                               sums of v and v*x there and a finalize kernel derives col_sum/col_sq/samp_sum/samp_sq from them. */
} cvb_gemm_args;
CVB_API int cvb_pw_gemm(const cvb_gemm_args* args, cvb_stream_t stream);
/* Two kernels implement cvb_pw_gemm (and two cvb_pw_wgrad): warp-specialised wgmma/TMA kernels (N >= 96 resp. K % 64 == 0)
 * and mma.sync kernels (narrow / odd shapes).  Testing hook: disable (0) / enable (1) the wgmma kernels so the two can be compared
 * on identical inputs; returns the previous setting. */
CVB_API int cvb_set_tc_enabled(int on);
/* Every kernel is launched with programmatic dependent launch (its set-up overlaps the previous kernel's tail; the kernel
 * itself orders its data accesses with griddepcontrol.wait).  Testing hook: plain stream-ordered launches (0) / PDL (1);
 * returns the previous setting. */
CVB_API int cvb_set_pdl_enabled(int on);

/* Weight gradient of a pointwise conv / linear:  dW[N,K] += sum_m load(G)[m,n] * load(A)[m,k];  dbias[n] += sum_m load(G)[m,n]
 * (autograd of F.conv2d / F.linear at the call sites above).  G modes: RAW or BNB; A modes: RAW/AFF/AFF_SILU/SILU/GN. */
typedef struct {
  int M, N, K;
  const void* G; int ldg; const void* G2; int ldg2; int g_mode;
  const float* g_p0; const float* g_p1; const float* g_p2; /* per-N */
  const void* A; int lda; int a_mode;
  const float* a_p0; const float* a_p1;                    /* per-K */
  const float* row_mean; const float* row_rstd; int rows_per_sample;
  float* dW; int lddw; /* fp32 [N, lddw], accumulated (+=): caller zeroes */
  float* dbias;        /* fp32 [N] or NULL, accumulated (+=) */
} cvb_wgrad_args;
CVB_API int cvb_pw_wgrad(const cvb_wgrad_args* args, cvb_stream_t stream);

/* OUT[m,k] = load(A[,A2])[m,k] (bf16): materialises one of the operand load modes above.  Used for WIDE layers (K >= 384 with
 * several N tiles, all late-stage and L2-resident) where applying the prologue once is cheaper than once per N tile.
 * K <= 8192, M < 2^31. */
CVB_API int cvb_apply_load_mode(const void* A, int lda, const void* A2, int lda2, int mode, const float* p0, const float* p1, const float* p2,
                                const float* row_mean, const float* row_rstd, int rows_per_sample, void* OUT, int ldo, int64_t M, int K,
                                cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Depthwise 3x3 convolution, pad = dilation, stride 1|2, NHWC (ConvLayer2d(groups=C): mobilenetv2.py:194-207,
 * mobilevit_block.py:369-379), and the undilated 5x5 one, pad 2, stride 1|2 (EfficientNet's MBConv blocks: cvnets/modules/efficientnet.py,
 * config/efficientnet.py).  dilation 0 / 1 = dense stencil (TMA walk kernels); dilation > 1 (stride 1 only) = the segmentation
 * backbones' output_stride 8 / 16 variants (base_image_encoder.py:38-47, mobilevit_v2.py:176-191), a direct-gather kernel.  The producer's BN(+SiLU) is applied on load (x_mode RAW/AFF/AFF_SILU); zero padding
 * is applied AFTER that transform, as in the reference where padding acts on the activated tensor.
 * Output: pre-BN y (bf16) + fp64 per-channel sum / sum of squares of the stored values.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct {
  int B, H, W, C, stride;
  const void* X; int x_mode; const float* x_p0; const float* x_p1;
  const float* Wt;  /* fp32 [K*K][C] (tap-major), values already rounded to bf16 (autocast semantics) */
  void* Y;          /* bf16 [B,Ho,Wo,C] */
  double* col_sum; double* col_sq;
  int dilation;     /* 0 or 1: none */
  int ksize;        /* K: 0 or 3 = 3x3, 5 = 5x5 (pad 2; dilation must be 0 / 1) */
} cvb_dw_fwd_args;
CVB_API int cvb_dw_fwd(const cvb_dw_fwd_args* args, cvb_stream_t stream);

/* Backward of the above, fused: dy = load(DZ[,Y2]) (RAW or BNB), dX = conv_transpose(dy) then through the producer's
 * activation (x_mode AFF_SILU: dX *= silu'(p0*x+p1)), statistics col_sum += dX, col_sq += dX*x for the producer's BN
 * backward, and dWt[K*K][C] += sum dy * load(X)(shifted).  Stride 2 needs even H and W. */
typedef struct {
  int B, H, W, C, stride;
  const void* DZ; const void* Y2; int g_mode; const float* g_p0; const float* g_p1; const float* g_p2;
  const void* X; int x_mode; const float* x_p0; const float* x_p1;
  const float* Wt;
  void* DX;         /* bf16 [B,H,W,C] */
  double* col_sum; double* col_sq; /* may be NULL when x_mode == RAW */
  float* dWt;       /* fp32 [K*K][C], accumulated (+=) */
  int dilation;     /* 0 or 1: none */
  int ksize;        /* as in cvb_dw_fwd_args */
} cvb_dw_bwd_args;
CVB_API int cvb_dw_bwd(const cvb_dw_bwd_args* args, cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Stem: the dense 3x3 stride-2 conv 3 -> C0 of MobileViTv2 (mobilevit_v2.py:37-45) runs as im2col + cvb_pw_gemm:
 * A[(b,oh,ow), ci*9+u*3+v] = bf16(X[b,ci,2oh+u-1,2ow+v-1]) (zero padded; columns 27..31 are zero), fp32 image in with
 * arbitrary element strides (NCHW or channels_last).  The 32-column bf16 patch matrix costs 64 B/pixel (the stem's
 * output alone is 64 B/pixel at C0=32) and lets forward, BN statistics and dW reuse the GEMM kernels.
 * The gather folds in the reference's batch-mixing input transforms (SURVEY.md 8f row 3: engine/training_engine.py:236-238,
 * data/transforms/image_torch.py:99-137 RandomMixup, :290-342 RandomCutmix).  mix: DEVICE float[6] = {mode, lambda, x1, y1, x2, y2} or NULL;
 * every sample pairs with its predecessor in the batch (image.roll(1, 0)): mode 1 (mixup) x = lambda*x + (1-lambda)*x_prev in fp32;
 * mode 2 (cutmix) rows [y1,y2) x columns [x1,x2) come from x_prev; mode 0 or NULL = off.  The matching target distribution
 * lambda*onehot(y[b]) + (1-lambda)*onehot(y[b-1]) is what cvb_ce_fwd / cvb_ce_bwd use when given the same `mix`.
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_stem_im2col(const float* X, int64_t sxn, int64_t sxc, int64_t sxh, int64_t sxw, int B, int H, int W, void* A, const float* mix,
                    cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * BatchNorm2d bookkeeping (cvnets/layers/normalization/batch_norm.py:14-49; math SURVEY App. A1)
 * ------------------------------------------------------------------------------------------------------------- */
/* training: from fp64 sum / sumsq over `count` values per channel -> mean, rstd, scale=gamma*rstd, shift=beta-mean*scale;
 * running_mean/var EMA (unbiased var) if running_mean != NULL; num_batches_tracked += 1 if not NULL. */
CVB_API int cvb_bn_finalize(const double* sum, const double* sq, double count, const float* gamma, const float* beta, float eps,
                    float momentum, float* running_mean, float* running_var, int64_t* num_batches_tracked,
                    float* mean, float* rstd, float* scale, float* shift, int C, cvb_stream_t stream);
/* eval: scale/shift from running statistics */
CVB_API int cvb_bn_eval_scale_shift(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                            float eps, float* mean, float* rstd, float* scale, float* shift, int C, cvb_stream_t stream);
/* backward: from sum_dz, sum_dz_y -> dgamma, dbeta and the coefficients of dy = c1*dz + c2*y + c3.
 * eval_mode != 0: statistics were constants: c1 = gamma*rstd, c2 = c3 = 0. */
CVB_API int cvb_bn_bwd_finalize(const double* sum_dz, const double* sum_dzy, double count, const float* gamma, const float* mean,
                        const float* rstd, int eval_mode, float* dgamma, float* dbeta, float* c1, float* c2, float* c3,
                        int C, cvb_stream_t stream);
/* out = act(scale*y + shift) (+ R): materialises a module output.  act: 0 none, 1 silu. */
CVB_API int cvb_bn_apply(const void* Y, const float* scale, const float* shift, int act, const void* R, void* OUT, int64_t M, int C,
                 cvb_stream_t stream);
/* sum_dz[c] += dz, sum_dzy[c] += dz*y with dz = dout (act=0) or dout*silu'(scale*y+shift) (act=1); dz optionally stored */
CVB_API int cvb_bn_bwd_reduce(const void* DOUT, const void* Y, const float* scale, const float* shift, int act, void* DZ /* bf16 out or NULL */,
                      double* sum_dz, double* sum_dzy, int64_t M, int C, cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * GroupNorm(1, C) == layer_norm_2d bookkeeping (cvnets/layers/normalization/layer_norm.py:75-108; SURVEY App. A4)
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_gn_finalize(const double* samp_sum, const double* samp_sq, double count, float eps, float* mean, float* rstd, int B,
                    cvb_stream_t stream);
/* per-sample sum / sumsq of a bf16 [B*rows, C] tensor (used when no producer epilogue could emit them) */
CVB_API int cvb_gn_stats(const void* X, int ldx, int B, int rows_per_sample, int C, double* samp_sum, double* samp_sq, cvb_stream_t stream);
/* phase 2 of GroupNorm backward: dx = rstd[b]*(g - m1[b] - xh*m2[b]) + dres, m1 = sg/count, m2 = sgx/count;
 * optional col_sum[c] += dx (bias gradient of the layer that produced the residual stream). */
CVB_API int cvb_gn_bwd_apply(const void* G, const void* X, const float* mean, const float* rstd, const double* sg, const double* sgx,
                     double count, const void* DRES, void* DX, int B, int rows_per_sample, int C, double* col_sum,
                     cvb_stream_t stream);

/* Stand-alone GroupNorm(1, C) backward (autograd of F.group_norm as LayerNorm2D_NCHW calls it, layer_norm.py:105-108) in two launches:
 * V = gradient w.r.t. the normalised+affine output, X = the layer's input, mean/rstd per sample.  dgamma[c] += sum V*xhat, dbeta[c] += sum V
 * (fp64, caller zeroes), samp_ws: ZEROED fp64 [2][B] scratch; DX = rstd*(V*gamma - mean(V*gamma) - xhat*mean(V*gamma*xhat)) (+ DRES). */
CVB_API int cvb_gn_bwd(const void* V, const void* X, const float* mean, const float* rstd, const float* gamma, double count, const void* DRES,
               void* DX, int B, int rows_per_sample, int C, double* dgamma, double* dbeta, double* samp_ws, cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * LinearSelfAttention core between qkv_proj and out_proj (cvnets/layers/linear_attention.py:134-161; SURVEY App. A5),
 * with unfold/fold (mobilevit_block.py:526-555) collapsed into indexing: the feature map stays [B,H,W,*] and the four
 * pixel positions p of every 2x2 patch are the (row parity, column parity) sub-lattices.
 * QKV: bf16 [B*H*W, ldq] with columns [0,d)=key, [d,2d)=value, 2d=query (ldq >= 2d+8, multiple of 8).
 * fwd:  s = softmax over the N=(H/2)(W/2) patches of q;  ctx[c] = sum_n key*s;  O = relu(value)*ctx.
 * Saves s (fp32 [B,4,N]) and ctx (fp32 [B,4,d]) for the backward.
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_linattn_fwd(const void* QKV, int ldq, int B, int H, int W, int d, int patch, void* O, int ldo, float* S, float* CTX,
                    cvb_stream_t stream);
/* bwd: from dO -> dQKV (same layout as QKV; pad columns zeroed); dbias_qkv[2d+1 (+pad)] += column sums if not NULL */
CVB_API int cvb_linattn_bwd(const void* QKV, int ldq, const void* DO, int ldo, const float* S, const float* CTX, int B, int H, int W,
                    int d, int patch, void* DQKV, float* dbias, cvb_stream_t stream);
/* patch = 2: folded feature map as above.  patch = 0: the tensor is the UNFOLDED matrix [B, P = H, N = W, ld] itself, i.e. a stand-alone
 * LinearSelfAttention applied to a [B, d, P, N] input in channels-last memory (linear_attention.py:134-161, 209-215).
 * Cross-attention (LinearSelfAttention._forward_cross_attn, linear_attention.py:163-207; LinearAttnFFN cross branch transformer.py:254-260):
 * query + key come from the projection of x_prev (QK_prev: [B, P, M, ldq], columns as above), the values from the projection of x
 * (V_x: [B, P, N, ldv], value columns [d, 2d)); softmax / context over M, output O [B, P, N, ldo].  S: [B, P, M], CTX: [B, P, d].
 * bwd writes the key/query columns of DQK_prev and the value columns of DV_x (the caller zero-fills the other columns of both). */
CVB_API int cvb_linattn_cross_fwd(const void* QK_prev, int ldq, int B, int P, int M, int d, const void* V_x, int ldv, int N, void* O, int ldo,
                          float* S, float* CTX, cvb_stream_t stream);
CVB_API int cvb_linattn_cross_bwd(const void* QK_prev, int ldq, const void* V_x, int ldv, const void* DO, int ldo, const float* S, const float* CTX,
                          int B, int P, int M, int N, int d, void* DQK_prev, void* DV_x, float* dbias, cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * MultiHeadAttention core (cvnets/layers/multi_head_attention.py:135-239, self-attention branch) and LayerNorm statistics
 * (cvnets/layers/normalization/layer_norm.py:14-72: nn.LayerNorm over the last dimension of [N, S, C]).
 * QKV: bf16 [B*S, ldq] rows = tokens, columns [q (H*c) | k (H*c) | v (H*c)] exactly as qkv_proj writes them (:148-153);
 * O: bf16 [B*S, ldo] with head h at columns h*c.. (the layout out_proj reads, :236).  scale = head_dim^-0.5 (:70, :187).
 * attn_mask: fp32 [B, S, S] additive (or NULL, :197-208); key_padding_mask: uint8 [B, S], non-zero = masked with -inf (:210-224).
 * Softmax in fp32 (:226-228).  LSE: fp32 [B, H, S] log-sum-exp (base 2) saved for the backward.  Even c <= 64; S <= 256, or any S for c = 64.
 * head_dim == 64 (ViT-B / CLIP image tower, key-padding masks included) runs on wgmma tensor cores: S <= 256 in mha_tc.cu (TMA-staged operands,
 * whole score rows in registers), S > 256 (ViT / CLIP at 256-512 px crops) in mha_long.cu (K/V and Q/dO streamed through shared memory in
 * 64-row tiles, online softmax; a backward without atomics, bitwise reproducible).  Every other head_dim, and heads with an additive mask at
 * S <= 256, run on the mma.sync kernels (mha.cu).
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_mha_fwd(const void* QKV, int ldq, int B, int S, int H, int head_dim, float scale, const float* attn_mask,
                const unsigned char* key_padding_mask, void* O, int ldo, float* LSE, cvb_stream_t stream);
/* dQKV (bf16 [B*S, lddq], same column layout as QKV) from dO; recomputes the probabilities from LSE. */
CVB_API int cvb_mha_bwd(const void* QKV, int ldq, const void* O, const void* DO, int ldo, const float* LSE, int B, int S, int H, int head_dim,
                float scale, const float* attn_mask, const unsigned char* key_padding_mask, void* DQKV, int lddq, cvb_stream_t stream);
/* Testing hook: which kernel family serves a head, forward and backward alike.  0 = automatic (default, as described above);
 * 1 = the mma.sync kernels wherever they can run (S <= 256); 2 = the streaming kernels for every head_dim-64 shape.  Modes 1 and 2
 * cross-check the families against each other; any other value selects 0.  Returns the previous mode. */
CVB_API int cvb_set_mha_impl(int mode);
/* per-token LayerNorm statistics of a bf16 [M, C] matrix: mean[m], rstd[m] = 1/sqrt(var + eps) (biased variance, fp32 math like
 * nn.LayerNorm under autocast).  The normalisation itself is the GN load mode of the consuming GEMM with rows_per_sample = 1. */
/* LayerNorm backward of a [M, C] token matrix in one pass (autograd of nn.LayerNorm as used at transformer.py:77-95):
 * V = gradient w.r.t. the LayerNorm OUTPUT (bf16), X = its input, mean/rstd from cvb_ln_stats or cvb_gn_finalize(count = C);
 * DX = rstd * (V*gamma - mean_c(V*gamma) - xhat * mean_c(V*gamma*xhat)) + DRES (optional residual-stream gradient);
 * dgamma[c] += sum_m V*xhat, dbeta[c] += sum_m V, col_sum[c] += sum_m DX (optional: bias gradient of the producer).  C <= 1280. */
CVB_API int cvb_ln_bwd(const void* V, const void* X, const float* mean, const float* rstd, const float* gamma, const void* DRES, void* DX,
               int64_t M, int C, double* dgamma, double* dbeta, double* col_sum, cvb_stream_t stream);
/* element-wise activation passes over contiguous bf16 tensors of n elements (n % 8 == 0): Y = act(X);  DX = DY * act'(X), act = kind.
 * Used by the TransformerEncoder FFN (cvnets/modules/transformer.py:86-95) when the activation is not the GEMM-fused SiLU, and by
 * InvertedResidualSE / SqueezeExcitation. */
enum {
  CVB_ACT_SILU = 0,     /* cvnets/layers/activation/swish.py                      */
  CVB_ACT_GELU,         /* cvnets/layers/activation/gelu.py: nn.GELU, erf form    */
  CVB_ACT_RELU,         /* cvnets/layers/activation/relu.py                       */
  CVB_ACT_HARDSWISH,    /* cvnets/layers/activation/hard_swish.py: x*relu6(x+3)/6 */
  CVB_ACT_HARDSIGMOID,  /* cvnets/layers/activation/hard_sigmoid.py: relu6(x+3)/6 */
  CVB_ACT_SIGMOID       /* cvnets/layers/activation/sigmoid.py                    */
};
CVB_API int cvb_act_fwd(const void* X, void* Y, int64_t n, int kind, cvb_stream_t stream);
CVB_API int cvb_act_bwd(const void* DY, const void* X, void* DX, int64_t n, int kind, cvb_stream_t stream);
CVB_API int cvb_ln_stats(const void* X, int ldx, int64_t M, int C, float eps, float* mean, float* rstd, cvb_stream_t stream);
/* Squeeze-excitation channel scaling (cvnets/modules/squeeze_excitation.py:82-83, used by InvertedResidualSE, cvnets/modules/mobilenetv2.py:16-138):
 * Y[b,p,c] = X[b,p,c] * S[b,c] on a channels-last bf16 map [B, HW, C] with the bf16 scale vector S [B, C] (C % 8 == 0);
 * backward: DX = DY * S and DS[b,c] += sum_p DY * X (fp32, zero-initialised by the caller; the partial sums meet in an fp64 scratch, so DS
 * is the same bits run to run). */
CVB_API int cvb_se_scale_fwd(const void* X, const void* S, void* Y, int B, int HW, int C, cvb_stream_t stream);
CVB_API int cvb_se_scale_bwd(const void* DY, const void* X, const void* S, void* DX, float* DS, int B, int HW, int C, cvb_stream_t stream);
/* Dropout (cvnets/layers/dropout.py == nn.Dropout) and stochastic depth (torchvision.ops.StochasticDepth(mode="row"), cvnets/modules/transformer.py:97-100)
 * folded into the residual add of the transformer blocks (transformer.py:139-156) on bf16 [M, C] matrices (C % 8 == 0):
 *   fwd: Y = R + V * e * r   (R optional),   bwd: DV = DY * e * r;   e ~ Bernoulli(1-p)/(1-p) per element, r ~ Bernoulli(1-p_row)/(1-p_row) per
 *   sample (rows_per_sample consecutive rows).  The masks are a counter-based hash of the 64-bit key at `key` (device memory) -- never stored; the
 *   backward passes the forward's key.  cvb_rng_next draws a key from the device-resident state {seed, counter} (2 x uint64) and advances the
 *   counter on the device, so a captured CUDA graph draws fresh masks at every replay. */
CVB_API int cvb_rng_next(void* state, void* key_out, cvb_stream_t stream);
CVB_API int cvb_dropout_fwd(const void* V, const void* R, void* Y, int64_t M, int C, int rows_per_sample, float p, float p_row, const void* key,
                    cvb_stream_t stream);
CVB_API int cvb_dropout_bwd(const void* DY, void* DV, int64_t M, int C, int rows_per_sample, float p, float p_row, const void* key, cvb_stream_t stream);

/* RangeAugment (cvnets/neural_augmentor/neural_aug.py DistributionNeuralAugmentor, loss_fn/neural_augmentation.py) on fp32 NCHW images [B, 3, H, W]
 * in [0, 1], contiguous.  `mix` (NULL = off) is the batch-mixing record of cvb_stem_im2col, applied on the fly: the augmentor sees the mixed image.
 * Every augmentation is affine per (sample, channel), so the chain is x_aug = clip(A x_mix + Bc + C eps, 0, 1) with coef[b, c] = (A, Bc, C).
 * Draws are hashes of the 64-bit key at `key` (cvb_rng_next), recomputed by every kernel that needs them:
 *   cvb_na_plan     draw table tab[4 + 3 B]: tab[0..2] augmentation (0 brightness, 1 contrast, 2 noise) at each position of a uniformly random
 *                   order of the enabled ones (bit k of `enabled`; -1 past them), tab[3] their count, tab[4 + k B + b] = u ~ U[0, 1) if sample b is
 *                   one of the max(1, B / 2) distinct samples drawn for augmentation k, else -1.  B <= 4096.
 *   cvb_na_noise    the N(0, 1) field eps [B, 3, H, W] the other kernels recompute (for tests).
 *   cvb_na_stats    per-plane means of x_mix and eps (fp64 [B * 3] each; eps only when need_eps).
 *   cvb_na_compose  coef fp32 [B * 3, 3] from the table, the means and the sampler parameters raw[6] = (_low, _high) of brightness, contrast,
 *                   noise (device fp32 scalars; NULL pairs = disabled): low / high = sigmoid(raw) (max - min) + min with the reference's bounds.
 *   cvb_na_apply    Y = x_aug (fp32 NCHW) and sq[b * 3 + c] = sum (x_aug - x_mix)^2 (fp64).
 *   cvb_na_bwd_reduce  red[b * 3 + c] = (sum g x_mix, sum g, sum g eps) of g = [0 <= pre-clip <= 1] (DY + 2 g_sq (x_aug - x_mix)) (DY or g_sq NULL = 0).
 *   cvb_na_param_grad  grads[j] = d loss / d raw[j] (fp32 scalars, overwritten) from red: the chain rule through the composition, the draws, the
 *                   contrast means and the sigmoid bounds.
 *   cvb_na_loss_fwd loss = w_na * L_na + w_ce * *ce (the composite loss; ce may be NULL = 0), L_na = alpha / 65025 * mean_b smooth_l1(mse_b -
 *                   target[min(step, T - 1)]), mse_b = 65025 * sum_c sq[b, c] / (3 H W); parts (may be NULL) = (*ce, L_na).
 *   cvb_na_loss_bwd g_sq[b * 3 + c] = d loss / d sq[b, c], times *grad_out and *grad_scale (either may be NULL = 1); g_ce (may be NULL) =
 *                   *grad_out * w_ce, the gradient handed to the cross entropy (whose backward applies the loss scale).
 * All sums are fp64 in a fixed order: the same bits run to run. */
CVB_API int cvb_na_plan(const void* key, int B, int enabled, float* tab, cvb_stream_t stream);
CVB_API int cvb_na_noise(const void* key, int B, int H, int W, float* eps, cvb_stream_t stream);
CVB_API int cvb_na_stats(const float* X, const float* mix, const void* key, int B, int H, int W, int need_eps, double* mu_x, double* mu_e, cvb_stream_t stream);
CVB_API int cvb_na_compose(const float* tab, const double* mu_x, const double* mu_e, const float* const* raw, int B, float* coef, cvb_stream_t stream);
CVB_API int cvb_na_apply(const float* X, const float* mix, const void* key, const float* coef, int B, int H, int W, int need_eps, float* Y, double* sq,
                 cvb_stream_t stream);
CVB_API int cvb_na_bwd_reduce(const float* DY, const double* g_sq, const float* X, const float* mix, const void* key, const float* coef, int B, int H, int W,
                      int need_eps, double* red, cvb_stream_t stream);
CVB_API int cvb_na_param_grad(const float* tab, const double* mu_x, const double* mu_e, const double* red, const float* const* raw, int B,
                      float* const* grads, cvb_stream_t stream);
CVB_API int cvb_na_loss_fwd(const double* sq, int B, int H, int W, const float* target, int T, const int64_t* step, float alpha, float w_na, const float* ce,
                    float w_ce, float* loss, float* parts, cvb_stream_t stream);
CVB_API int cvb_na_loss_bwd(const double* sq, int B, int H, int W, const float* target, int T, const int64_t* step, float alpha, float w_na,
                    const float* grad_out, const float* grad_scale, double* g_sq, float* g_ce, float w_ce, cvb_stream_t stream);
/* Input gradient of the stem conv (3 -> C0, 3x3, stride 2, pad 1): dX fp32 NCHW [B, 3, 2 Ho, 2 Wo] = conv_transpose(dy, W) with
 * dy = bf16(p0 dz + p1 y + p2) (CVB_A_BNB on the bf16 [B*Ho*Wo, C0] dz / y, coef fp32 [3, C0]) and the prepared bf16 weight [C0, 32]
 * (columns ci*9 + u*3 + v).  C0 a multiple of 8, <= 64. */
CVB_API int cvb_stem_dgrad(const void* dz, const void* y, const float* coef, const void* w, int B, int Ho, int Wo, int C0, float* dX, cvb_stream_t stream);
/* Input gradient of the ViT / CLIP conv stem's first conv (3 -> C0, 4x4, stride 4, pad 1; vit.py:90-121): dX fp32 NCHW [B, 3, 4 Ho, 4 Wo] =
 * conv_transpose(dy, W) with dy = bf16(p0 dz + p1 y + p2) (CVB_A_BNB on the bf16 [B*Ho*Wo, C0] dz / y, coef fp32 [3, C0]) and the prepared
 * bf16 weight [C0, 48] (CVB_PREP_PATCH: columns (u*4 + v)*3 + ci).  Every element of dX is written, the last image row and column (which
 * lie in no window) with 0; no atomics, bitwise reproducible.  C0 a multiple of 16, <= 320; dz, y, coef, dX 16-byte aligned. */
CVB_API int cvb_patch_stem_dgrad(const void* dz, const void* y, const float* coef, const void* w, int B, int Ho, int Wo, int C0, float* dX,
                                 cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Per-step tail of the training loop (engine/training_engine.py:289-312) on FLAT fp32 buffers of n elements: GradScaler unscale +
 * inf check, clip_grad_norm_, AdamW, GradScaler update -- two launches, all state on the device (CUDA-graph friendly).
 *   stats : fp32[4], zero-initialised once; [0] sum of squares of the unscaled gradients, [1] # non-finite elements,
 *           [2] 1/scale used by this step, [3] internal block counter (the step kernel clears [0], [1], [3] when it is done)
 *   scale : fp32[2] = {loss scale, growth tracker}   (torch.amp.GradScaler: init 65536, growth 2.0, backoff 0.5, interval 2000)
 *   step  : fp32[1] optimizer step count
 * cvb_grad_norm must precede cvb_adamw_step.  AdamW follows torch.optim.AdamW exactly (decoupled weight decay p *= 1 - lr*wd[i],
 * bias-corrected moments, eps added after the sqrt); weight_decay is per ELEMENT so the reference's two parameter groups
 * (cvnets/misc/common.py:122-176: 1-D parameters are not decayed) need no segment table.  max_norm <= 0 disables clipping.
 * hp    : fp32[1] DEVICE scalar = learning rate (written by the scheduler each iteration: scheduler.update_lr, training_engine.py:246-249)
 * grad_div : gradients are divided by loss_scale * grad_div (DDP's mean over ranks: grad_div = world size, main_train.py:90-96)
 * ema / ema_momentum : optional fp32[n] moving average updated in the same pass, ema = ema*(1-momentum) + momentum*param
 *           (cvnets/misc/averaging_utils.py:43-55; also on skipped steps, like the reference's per-iteration update); NULL = off
 * partials : fp32[2 * cvb_grad_norm_blocks(n)] scratch: per-block (sum of squares, non-finite count), combined in a fixed order by the step
 *           kernel so that the norm / clip coefficient / update are bit-identical on every data-parallel rank
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_grad_norm_blocks(int64_t n);
CVB_API int cvb_grad_norm(const float* grads, int64_t n, const float* scale, float grad_div, float* stats, float* partials, cvb_stream_t stream);
CVB_API int cvb_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const float* weight_decay, int64_t n,
                   const float* hp, float beta1, float beta2, float eps, float max_norm, float* stats, float* scale, float* step,
                   float growth_factor, float backoff_factor, int growth_interval, float* ema, float ema_momentum, const float* partials,
                   cvb_stream_t stream);
/* The same step with torch.optim.SGD(momentum, dampening=0, nesterov, weight_decay) in place of AdamW (the SGD recipes: EfficientNet,
 * MobileNet v1-v3): g' = g*unscale*clip + weight_decay[i]*p;  momentum_buf = momentum*momentum_buf + g' (zero-initialised, which equals
 * torch's first-step clone);  p -= lr * (g' + momentum*momentum_buf) with nesterov != 0, lr * momentum_buf without.  Same stats / scale /
 * step / EMA / partials semantics as cvb_adamw_step; cvb_grad_norm must precede it. */
CVB_API int cvb_sgd_step(float* params, const float* grads, float* momentum_buf, const float* weight_decay, int64_t n, const float* hp, float momentum,
                         int nesterov, float max_norm, float* stats, float* scale, float* step, float growth_factor, float backoff_factor,
                         int growth_interval, float* ema, float ema_momentum, const float* partials, cvb_stream_t stream);
/* Gradient accumulation over micro-batches (engine/training_engine.py:286-312 with common.accum_freq > 1: gradients are SUMMED, the loss is
 * not divided): acc[i] += g[i] over n fp32 elements, one IEEE add per element (round to nearest, subnormals kept), so the result is bitwise
 * torch's fp32 add.  acc and g 16-byte aligned; grid of min(ceil(n / 1024), 4 * SMs) CTAs of 256 threads, grid-stride. */
CVB_API int cvb_grad_accumulate(float* acc, const float* g, int64_t n, cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Classification loss of the step: F.cross_entropy(prediction, target, ignore_index, label_smoothing), mean over the non-ignored
 * rows (loss_fn/classification/cross_entropy.py:74-95).  logits: bf16 [B, ld] (C valid columns); target: int64 [B].
 * fwd: lse fp32[B] (saved), loss fp32[1], n_valid fp32[1].   bwd: dlogits bf16 [B, ldd] (columns >= C zeroed) =
 * grad_out * grad_scale * (softmax - smoothed one-hot) / n_valid; grad_out / grad_scale are DEVICE scalars or NULL (= 1): the
 * GradScaler's loss scale (engine/training_engine.py:287) multiplies here instead of in a separate kernel.
 * logit_scale (DEVICE scalar or NULL): CLIP's learnable temperature (cvnets/models/multi_modal_img_text/clip.py: logit_scale.exp().clamp(0, 100);
 * loss_fn/multi_modal_img_text/contrastive_loss_clip.py:74-79): the rows are RAW similarities and the loss is taken of s * raw; bwd returns the
 * gradient w.r.t. the raw similarities and accumulates d loss / d logit_scale into dlogit_scale (fp32, atomically; 0 where the clamp is active).
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_ce_fwd(const void* logits, int ld, int B, int C, const int64_t* target, int ignore_index, float label_smoothing, float* lse,
               float* loss, float* n_valid, const float* mix /* see cvb_stem_im2col; NULL = plain targets */, const float* logit_scale,
               cvb_stream_t stream);
CVB_API int cvb_ce_bwd(const void* logits, int ld, int B, int C, const int64_t* target, int ignore_index, float label_smoothing, const float* lse,
               const float* n_valid, const float* grad_out, const float* grad_scale, void* dlogits, int ldd, const float* mix,
               const float* logit_scale, float* dlogit_scale, cvb_stream_t stream);

/* Batched fp64 -> fp32 scatter: dst[i] = (float)src[i] for every descriptor (one launch per module backward: the fp64 statistics
 * accumulators that ARE gradients -- GroupNorm dgamma/dbeta, bias gradients -- go straight into the flat gradient buffer). */
typedef struct {
  const double* src; float* dst; int n; int pad;
} cvb_cast_desc;
CVB_API int cvb_cast_f64_f32(const cvb_cast_desc* descs_device, int n_desc, int max_n, cvb_stream_t stream);
/* ---------------------------------------------------------------------------------------------------------------
 * CLIP text tower edges and feature normalisation (BASELINE.json configs[4]; csrc/clip.cu)
 *   embedding: out[b,s,:] = bf16(table[tokens[b,s],:] + pos[s,:])  (cvnets/text_encoders/transformer.py:328-341); bwd: dtable[token] += dout
 *              (fp32 atomics), dpos[s] += sum_b dout[b,s]
 *   eot gather: out[b,:] = X[b, argmax_s tokens[b,s], :] (transformer.py:413-421); idx[b] saved; bwd scatters into a zero-filled dX
 *   l2norm: Y = X / max(||X||_2, eps) per row (F.normalize, transformer.py:423-425); inv_norm saved; bwd dx = inv*(dy - y (y.dy))
 *   transpose / add: Y[c,r] = X[r,c];  OUT = bf16(A + B) (A bf16 or NULL, B fp32) -- glue of the contrastive loss's gradient assembly
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_embedding_fwd(const int64_t* tokens, const float* table, const float* pos, void* out, int B, int S, int C, int V, cvb_stream_t stream);
CVB_API int cvb_embedding_bwd(const void* dout, const int64_t* tokens, float* dtable, float* dpos, int B, int S, int C, int V, cvb_stream_t stream);
CVB_API int cvb_eot_gather_fwd(const void* X, const int64_t* tokens, int B, int S, int C, void* out, int* idx, cvb_stream_t stream);
CVB_API int cvb_eot_gather_bwd(const void* dout, const int* idx, int B, int S, int C, void* dX, cvb_stream_t stream);
CVB_API int cvb_l2norm_fwd(const void* X, void* Y, float* inv_norm, int M, int C, float eps, cvb_stream_t stream);
CVB_API int cvb_l2norm_bwd(const void* DY, const void* Y, const float* inv_norm, void* DX, int M, int C, cvb_stream_t stream);
CVB_API int cvb_transpose_bf16(const void* X, void* Y, int R, int C, cvb_stream_t stream);
CVB_API int cvb_add_bf16_f32(const void* A, const float* B, void* OUT, int64_t n, cvb_stream_t stream);
/* ---------------------------------------------------------------------------------------------------------------
 * CLIP zero-shot evaluation (cvnets/text_encoders/transformer.py:428-504, cvnets/models/multi_modal_img_text/clip.py:171-202,
 * metrics/topk_accuracy.py; csrc/zeroshot.cu)
 *   class embedding: X = bf16 [R, ldx] projected caption features BEFORE normalisation; perm[c*M + m] = the row of caption m of class c
 *              (rows outside [0, R) are skipped).  table[k*Cl + c] = normalize(mean_m normalize(X[perm[c*M + m]])), all in fp32, with
 *              F.normalize's x / max(||x||, 1e-12) and the captions added in order m = 0..M-1.  One writer per class, no atomics:
 *              bitwise reproducible.  d % 8 == 0, d <= 1024.
 *   logits / top-k: img = bf16 [B, ldi] L2-normalised image features, table fp32 [d, Cl]; logits fp32 [B, Cl] = scale * img @ table (or
 *              NULL).  With targets (int64 [B]) and hits (int64 [2]) given, the rank of a row is the number of classes whose logit is
 *              strictly greater than the target's; hits[0] += (rank < 1), hits[1] += (rank < 5).  A target outside [0, Cl) is a miss.
 *              Integer adds only: the counts do not depend on the order of the CTAs.  No host sync.
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_zs_class_embed(const void* X, int ldx, int R, const int* perm, int Cl, int M, int d, float* table, cvb_stream_t stream);
CVB_API int cvb_zs_logits_topk(const void* img, int ldi, const float* table, int B, int d, int Cl, float scale, const int64_t* targets,
                               float* logits, int64_t* hits, cvb_stream_t stream);
/* ---------------------------------------------------------------------------------------------------------------
 * Validation of the classification recipes (engine/training_engine.py:val_epoch: loss, top1, top5; csrc/metrics.cu)
 *   cls metrics: logits bf16 [B, ld] (C valid columns, C >= 1), target int64 [B].  Per row whose target is not ignore_index: the cross
 *              entropy log-sum-exp - logit[target] WITHOUT label smoothing (the reference's loss in eval mode), and the rank of the
 *              target = the number of classes whose bf16 logit is STRICTLY greater than the target's; a row is a top-k hit iff rank < k
 *              (ties at the k-th place count for the target; C < 5 makes every counted row a top-5 hit).  A target outside [0, C) that is
 *              not ignore_index is a counted miss with a NaN loss.  Adds into device accumulators: loss_sum fp64[1] += sum of the
 *              per-row losses, counts int64[3] += {top-1 hits, top-5 hits, counted rows}.  row_loss: fp32 [B] scratch; ticket: int[1]
 *              scratch, zero before the first call (every call leaves it zero).  Bitwise deterministic: integer atomics, and the sum folds
 *              the fp32 row losses into fp64 in an order fixed by the row index alone.  No allocation, no host sync: capturable.
 *   EMA update: ema[i] = ema[i] * (1 - momentum) + momentum * src[i] over n fp32 elements, in the reference's operation order
 *              (cvnets/misc/averaging_utils.py:55: two rounded fp32 products, one rounded sum; 1 - momentum formed in double and rounded
 *              to fp32).  The EMA of the BatchNorm running statistics, one launch per training step.
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_cls_metrics(const void* logits, int ld, int B, int C, const int64_t* target, int ignore_index, double* loss_sum, int64_t* counts,
                            float* row_loss, int* ticket, cvb_stream_t stream);
CVB_API int cvb_ema_update(float* ema, const float* src, int64_t n, double momentum, cvb_stream_t stream);
/* cudaMemsetAsync(ptr, 0, bytes): the step's ONE workspace clear (a memset node under graph capture, not a kernel) */
CVB_API int cvb_memset_zero(void* ptr, int64_t bytes, cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * GlobalPool(mean) (cvnets/layers/global_pool.py:60-71)
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_global_pool_fwd(const void* X, int B, int HW, int C, void* OUT, cvb_stream_t stream);  /* bf16 -> bf16 [B,C] */
CVB_API int cvb_global_pool_bwd(const void* DOUT, int B, int HW, int C, void* DX, cvb_stream_t stream); /* broadcast / HW */

/* Layout kinds of cvb_prep_weights (fp32 parameter -> kernel layout) and of cvb_unprep_grad (fp32 gradient in a kernel layout -> the
 * parameter's layout; ROWMAJOR, TAPMAJOR_F32, VECTOR_F32 and PATCH only).  perm(r) = (r + rot) % rows for r < rows (rot = 1 moves the
 * reference's leading query row of qkv_proj to the end; ROWMAJOR, TRANSPOSED, VECTOR_F32). */
enum {
  CVB_PREP_ROWMAJOR = 0,  /* prep:   dst[r*ldd + c] = bf16(src[perm(r)*cols + c])   (row-major [rows, cols] -> bf16 [rows, ldd], zero padded)
                             unprep: dst[perm(r)*cols + c] = src[r*lds + c]                                                        */
  CVB_PREP_TRANSPOSED,    /* prep:   dst[c*ldd + r] = bf16(src[perm(r)*cols + c])   (transposed: -> bf16 [cols, ldd])              */
  CVB_PREP_TAPMAJOR_F32,  /* prep:   dst_f32[c*rows + r] = float(bf16(src[r*cols + c]))   (depthwise / stem: [C, taps] -> fp32 [taps, C],
                                     bf16-rounded)
                             unprep: tap-major [taps, C] -> [C, taps]                                                              */
  CVB_PREP_VECTOR_F32,    /* prep:   dst_f32[r] = src[perm(r)]   (fp32 vector gather, e.g. permuted bias; cols = 1)
                             unprep: dst[perm(r)] = src[r]                                                                         */
  CVB_PREP_PATCH,         /* prep:   dst[r*ldd + (t*Cin + ci)] = bf16(src[r*cols + ci*taps + t])   (dense conv weight [Cout, Cin, k, k] ->
                                     patch-matrix order; rot = taps = k*k)
                             unprep: dst[r*cols + ci*taps + t] = src[r*lds + t*Cin + ci], rot = taps (dense-conv weight gradients)  */
  CVB_PREP_PATCH_T        /* prep:   the same, transposed: dst[(t*Cin + ci)*ldd + r]                                                */
};

/* Batched weight preparation: one launch converts every fp32 parameter the step needs into the kernel layouts. */
typedef struct {
  const float* src; void* dst; int rows, cols, ldd, dst_rows; int kind; int rot;
} cvb_prep_desc;
CVB_API int cvb_prep_weights(const cvb_prep_desc* descs_device, int n_desc, int max_elems, cvb_stream_t stream);

/* fp32 gradient scatter-back for permuted layouts (qkv / depthwise / stem / dense-conv weight gradients). */
CVB_API int cvb_unprep_grad(const float* src, float* dst, int rows, int cols, int lds, int kind, int rot, cvb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Dense (groups = 1) k x k convolution = im2col + cvb_pw_gemm (ConvLayer2d at cvnets/models/classification/vit.py:90-121 -- the ViT / CLIP
 * conv stem -- and cvnets/modules/mobilevit_block.py:86-131 -- MobileViT-v1's 3x3 convs).  A[(b,i,j), (u*k+v)*Cin + ci] =
 * X[b, i*stride+u-pad, j*stride+v-pad, ci], zero outside the image and in the pad columns [k*k*Cin, lda).  X: fp32 or bf16 with arbitrary
 * ELEMENT strides (sxn, sxc, sxh, sxw) -- NCHW images as well as channels-last feature maps.  cvb_col2im is the adjoint for channels-last
 * bf16 gradients (a gather: no atomics), Cin % 8 == 0.
 * ------------------------------------------------------------------------------------------------------------- */
CVB_API int cvb_im2col(const void* X, int x_fp32, int64_t sxn, int64_t sxc, int64_t sxh, int64_t sxw, int B, int Cin, int H, int W, int k, int stride,
               int pad, void* A, int lda, cvb_stream_t stream);
CVB_API int cvb_col2im(const void* dA, int lda, int B, int Cin, int H, int W, int k, int stride, int pad, void* dX, cvb_stream_t stream);
/* MobileViT-v1 unfolding / folding (cvnets/modules/mobilevit_block.py:186-267) as a row permutation of the channels-last matrix:
 * feature-map row (b, h, w) <-> token row (b*P + p, n), p = (h % ph)*pw + (w % pw), n = (h / ph)*(W / pw) + (w / pw), P = ph*pw.
 * inverse = 0: X is the feature map [B*H*W, C], OUT the token matrix [B*P, N, C]; inverse = 1: the other way (folding).  The permutation
 * is its own adjoint with the flag flipped.  H, W must be multiples of the patch (the bilinear resize branch, :191-200, is not implemented). */
CVB_API int cvb_patch_permute(const void* X, void* OUT, int B, int H, int W, int C, int patch_h, int patch_w, int inverse, cvb_stream_t stream);
/* OUT[m, :] = [A[m, :C1] | B[m, :C2]] (torch.cat((res, fm), dim=1) on channels-last maps, mobilevit_block.py:287) and the adjoint split */
CVB_API int cvb_concat2(const void* A, const void* B, int C1, int C2, int64_t M, void* OUT, cvb_stream_t stream);
CVB_API int cvb_split2(const void* G, int C1, int C2, int64_t M, void* DA, void* DB, cvb_stream_t stream);
/* ViT token assembly (vit.py:476-507): out[b,0] = cls (no positional term), out[b,1+n] = patch[b,n] + pos'[n]; patch bf16 [B*N, C] (the
 * channels-last output of the last stem conv IS token-major), pos fp32 [n_pos, C], cls fp32 [C] or NULL, out bf16 [B, N(+1), C].
 * pos' is the table resampled to N rows as F.interpolate(pos [1, 1, n_pos, C], size=(N, C), mode="bilinear", align_corners=False) does
 * (cvnets/layers/positional_embedding.py:90-95) -- a 1-D linear resample of the flattened patch index, the identity when N == n_pos
 * (224 x 224 inputs) -- computed inside the kernel in fp32 and added to the patch row with one bf16 rounding.
 * bwd: dpatch = dout[:, 1:], dcls += sum_b dout[:, 0], dpos [n_pos, C] += the transposed stencil applied to sum_b dout[:, 1:] (fp32,
 * accumulated into caller-zeroed buffers; a gather without atomics: bitwise reproducible). */
CVB_API int cvb_vit_tokens_interp_fwd(const void* patch, const float* pos, int n_pos, const float* cls, void* out, int B, int N, int C,
                                      cvb_stream_t stream);
CVB_API int cvb_vit_tokens_interp_bwd(const void* dout, void* dpatch, float* dpos, int n_pos, float* dcls, int B, int N, int C, cvb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CVNETS_B200_H_ */
