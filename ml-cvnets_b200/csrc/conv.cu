// Dense (groups = 1) k x k convolution as im2col + the pointwise GEMM, and the ViT token assembly (sm_90a).
//
// The MobileViTv2 path has exactly one dense k x k conv (the stem, cvb_stem_im2col).  The other hot-path models need a few more:
// the ViT / CLIP conv stem ("patch embedding": 4x4 s4 p1, 2x2 s2, 2x2 s2 -- cvnets/models/classification/vit.py:90-121) and
// MobileViT-v1's dense 3x3 convs (cvnets/modules/mobilevit_block.py:86-131).  All of them are <= 6 % of their model's MACs, so they
// reuse the GEMM kernels through a gathered patch matrix instead of getting an implicit-GEMM kernel of their own:
//   A[(b,i,j), (u*k+v)*Cin + ci] = X[b, i*s+u-pad, j*s+v-pad, ci]   (zero outside the image; columns >= k*k*Cin are zero)
// Backward: dA = dY W (GEMM), dX = col2im(dA) as a GATHER (every input pixel sums its <= ceil(k/s)^2 contributions: no atomics),
// dW = dY^T A (weight-gradient GEMM).  The weight is re-ordered [Cout, Cin, k, k] -> [Cout, (u,v,ci)] by cvb_prep_weights kind 4.
#include "common.cuh"

namespace {

constexpr int CNT = 256;

// generic element-wise gather (any element strides, fp32 or bf16 source): used for 3-channel images and odd channel counts
__global__ void __launch_bounds__(CNT) im2col_generic_kernel(const void* __restrict__ X, int x_fp32, int64_t sn, int64_t sc, int64_t sh, int64_t sw, int Cin,
                                                             int H, int W, int k, int s, int pad, int Ho, int Wo, bf16* __restrict__ A, int lda, int64_t M) {
  pdl_wait();
  pdl_trigger();
  const int kk = k * k * Cin;
  const int64_t total = M * lda;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int64_t row = idx / lda;
    const int col = (int)(idx % lda);
    float v = 0.f;
    if (col < kk) {
      const int ci = col % Cin, uv = col / Cin, u = uv / k, w_ = uv % k;
      const int j = (int)(row % Wo), i = (int)((row / Wo) % Ho);
      const int64_t b = row / ((int64_t)Wo * Ho);
      const int h = i * s + u - pad, w = j * s + w_ - pad;
      if (h >= 0 && h < H && w >= 0 && w < W) {
        const int64_t off = b * sn + ci * sc + h * sh + w * sw;
        v = x_fp32 ? static_cast<const float*>(X)[off] : __bfloat162float(static_cast<const bf16*>(X)[off]);
      }
    }
    A[idx] = __float2bfloat16_rn(v);
  }
}

// channels-last bf16 source, Cin % 8 == 0: 16-byte chunks
__global__ void __launch_bounds__(CNT) im2col_nhwc_kernel(const bf16* __restrict__ X, int Cin, int H, int W, int k, int s, int pad, int Ho, int Wo,
                                                          bf16* __restrict__ A, int lda, int64_t M) {
  pdl_wait();
  pdl_trigger();
  const int cg = Cin >> 3, per_row = k * k * cg;
  const int64_t total = M * per_row;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int64_t row = idx / per_row;
    const int r = (int)(idx % per_row);
    const int c8 = r % cg, uv = r / cg, u = uv / k, w_ = uv % k;
    const int j = (int)(row % Wo), i = (int)((row / Wo) % Ho);
    const int64_t b = row / ((int64_t)Wo * Ho);
    const int h = i * s + u - pad, w = j * s + w_ - pad;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (h >= 0 && h < H && w >= 0 && w < W) v = ldg16(X + ((b * H + h) * (int64_t)W + w) * Cin + c8 * 8);
    stg16(A + row * lda + (int64_t)uv * Cin + c8 * 8, v);
  }
}

// dX[b,h,w,:] = sum over (u,v) with (h+pad-u) % s == 0, (w+pad-v) % s == 0 of dA[(b,(h+pad-u)/s,(w+pad-v)/s), (u,v,:)]
__global__ void __launch_bounds__(CNT) col2im_nhwc_kernel(const bf16* __restrict__ dA, int lda, int Cin, int H, int W, int k, int s, int pad, int Ho,
                                                          int Wo, bf16* __restrict__ dX, int64_t npix) {
  pdl_wait();
  pdl_trigger();
  const int cg = Cin >> 3;
  const int64_t total = npix * cg;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int64_t pix = idx / cg;
    const int c8 = (int)(idx % cg);
    const int w = (int)(pix % W), h = (int)((pix / W) % H);
    const int64_t b = pix / ((int64_t)W * H);
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    for (int u = 0; u < k; ++u) {
      const int hn = h + pad - u;
      if (hn < 0 || hn % s) continue;
      const int i = hn / s;
      if (i >= Ho) continue;
      for (int v = 0; v < k; ++v) {
        const int wn = w + pad - v;
        if (wn < 0 || wn % s) continue;
        const int j = wn / s;
        if (j >= Wo) continue;
        float f[8];
        unpack8(ldg16(dA + ((b * Ho + i) * (int64_t)Wo + j) * lda + (int64_t)(u * k + v) * Cin + c8 * 8), f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += f[q];
      }
    }
    stg16(dX + pix * Cin + c8 * 8, pack8(acc));
  }
}

// ViT token assembly (vit.py:476-507), backward without the positional stencil:
// dpatch[b, n] = dout[b, 1 + n];  dpos[n] += sum_b dout[b, 1 + n];  dcls += sum_b dout[b, 0].  One thread per (token position, 8 channels).
__global__ void __launch_bounds__(CNT) vit_tokens_bwd_kernel(const bf16* __restrict__ dout, bf16* __restrict__ dpatch, float* __restrict__ dpos,
                                                             float* __restrict__ dcls, int B, int N, int C, int has_cls) {
  pdl_wait();
  pdl_trigger();
  const int cg = C >> 3, S = N + has_cls;
  const int64_t total = (int64_t)S * cg;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int c8 = (int)(idx % cg), t = (int)(idx / cg);
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    for (int b = 0; b < B; ++b) {
      const uint4 raw = ldg16(dout + ((int64_t)b * S + t) * C + c8 * 8);
      float f[8];
      unpack8(raw, f);
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[q] += f[q];
      if (!(has_cls && t == 0)) stg16(dpatch + ((int64_t)b * N + (t - has_cls)) * C + c8 * 8, raw);
    }
    float* dst = (has_cls && t == 0) ? dcls + c8 * 8 : dpos + (int64_t)(t - has_cls) * C + c8 * 8;
#pragma unroll
    for (int q = 0; q < 8; ++q) dst[q] += acc[q];
  }
}

// Interpolated positional embeddings (cvnets/layers/positional_embedding.py:90-95): the reference resizes the [1, 1, n_pos, C] table to
// (N, C) with F.interpolate(mode="bilinear", align_corners=False).  The C axis maps onto itself, so this is a 1-D linear resample of the
// flattened patch index (not a 2-D resample of the patch grid), with PyTorch's source-index rule: scale = n_pos / N,
// src = max(scale (s + 0.5) - 0.5, 0), i0 = floor(src), i1 = i0 + (i0 < n_pos - 1), lambda = src - i0.  Unfused roundings: the products
// are computed as PyTorch's CPU kernel does.
__device__ __forceinline__ void interp_src(int s, float scale, int n_pos, int& i0, int& i1, float& lam) {
  const float src = fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn((float)s, 0.5f)), 0.5f), 0.f);
  i0 = (int)src;
  i1 = i0 + (i0 < n_pos - 1 ? 1 : 0);
  lam = __fsub_rn(src, (float)i0);
}

// ViT token assembly (vit.py:476-507, no positional term on the cls token):
// out[b, 0] = cls;  out[b, 1 + s] = patch[b, s] + (1 - lambda_s) pos[i0_s] + lambda_s pos[i1_s], in fp32, rounded once to bf16.
// At N == n_pos (224 px) the stencil is the identity (scale 1, i0_s = s, lambda_s = 0): out = patch + pos.
__global__ void __launch_bounds__(CNT) vit_tokens_interp_fwd_kernel(const bf16* __restrict__ patch, const float* __restrict__ pos, int n_pos, float scale,
                                                                    const float* __restrict__ cls, bf16* __restrict__ out, int B, int N, int C, int has_cls) {
  pdl_wait();
  pdl_trigger();
  const int cg = C >> 3, S = N + has_cls;
  const int64_t total = (int64_t)B * S * cg;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int c8 = (int)(idx % cg);
    const int64_t tok = idx / cg;
    const int t = (int)(tok % S);
    const int64_t b = tok / S;
    float f[8];
    if (has_cls && t == 0) {
#pragma unroll
      for (int q = 0; q < 8; ++q) f[q] = cls[c8 * 8 + q];
    } else {
      const int n = t - has_cls;
      int i0, i1;
      float lam;
      interp_src(n, scale, n_pos, i0, i1, lam);
      const float w0 = __fsub_rn(1.f, lam);
      unpack8(ldg16(patch + (b * N + n) * C + c8 * 8), f);
#pragma unroll
      for (int q = 0; q < 8; ++q)
        f[q] += __fadd_rn(__fmul_rn(w0, pos[(int64_t)i0 * C + c8 * 8 + q]), __fmul_rn(lam, pos[(int64_t)i1 * C + c8 * 8 + q]));
    }
    stg16(out + tok * C + c8 * 8, pack8(f));
  }
}

// dpos[j] += sum over output tokens s (ascending) of (1 - lambda_s) [i0_s == j] g[s] + lambda_s [i1_s == j] g[s], g = the batch sum of dout
// (fp32 [N, C]).  A gather over the few tokens whose stencil touches table row j: one thread per (j, 8 channels), no atomics.
__global__ void __launch_bounds__(CNT) vit_pos_interp_bwd_kernel(const float* __restrict__ g, float* __restrict__ dpos, int n_pos, float scale, int N,
                                                                 int C) {
  pdl_wait();
  pdl_trigger();
  const int cg = C >> 3;
  const int64_t total = (int64_t)n_pos * cg;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int c8 = (int)(idx % cg), j = (int)(idx / cg);
    // tokens with i0 in {j - 1, j}: src in [j - 1, j + 1), i.e. s in ((j - 0.5) / scale - 0.5, (j + 1.5) / scale - 0.5), widened by 2
    const int s_lo = max(0, (int)((j - 1.0f) / scale) - 2), s_hi = min(N - 1, (int)((j + 2.0f) / scale) + 2);
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    for (int s = s_lo; s <= s_hi; ++s) {
      int i0, i1;
      float lam;
      interp_src(s, scale, n_pos, i0, i1, lam);
      if (i0 != j && i1 != j) continue;
      const float* gs = g + (int64_t)s * C + c8 * 8;
      if (i0 == j) {
        const float w0 = __fsub_rn(1.f, lam);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = __fadd_rn(acc[q], __fmul_rn(w0, gs[q]));
      }
      if (i1 == j) {
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = __fadd_rn(acc[q], __fmul_rn(lam, gs[q]));
      }
    }
    float* dst = dpos + (int64_t)j * C + c8 * 8;
#pragma unroll
    for (int q = 0; q < 8; ++q) dst[q] += acc[q];
  }
}

// MobileViT-v1 unfolding / folding (cvnets/modules/mobilevit_block.py:186-267) on channels-last rows: the feature map row (b, h, w) and the
// token row (b*P + p, n) with p = (h % ph) * pw + (w % pw), n = (h / ph) * (W / pw) + (w / pw) hold the same C values: a row permutation.
__global__ void __launch_bounds__(CNT) patch_permute_kernel(const bf16* __restrict__ X, bf16* __restrict__ OUT, int H, int W, int C, int ph, int pw,
                                                            int inverse, int64_t npix) {
  pdl_wait();
  pdl_trigger();
  const int cg = C >> 3, nw = W / pw, N = (H / ph) * nw, P = ph * pw;
  const int64_t total = npix * cg;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int64_t pix = idx / cg;
    const int c8 = (int)(idx % cg);
    const int w = (int)(pix % W), h = (int)((pix / W) % H);
    const int64_t b = pix / ((int64_t)W * H);
    const int p = (h % ph) * pw + (w % pw), n = (h / ph) * nw + (w / pw);
    const int64_t tok = (b * P + p) * N + n;
    if (inverse) stg16(OUT + pix * C + c8 * 8, ldg16(X + tok * C + c8 * 8));
    else stg16(OUT + tok * C + c8 * 8, ldg16(X + pix * C + c8 * 8));
  }
}

// channel concatenation of two channels-last matrices (torch.cat((res, fm), dim=1), mobilevit_block.py:287) and its adjoint
__global__ void __launch_bounds__(CNT) concat2_kernel(const bf16* __restrict__ A, const bf16* __restrict__ B, bf16* __restrict__ OUT, int C1, int C2,
                                                      int split, int64_t M, bf16* __restrict__ DA, bf16* __restrict__ DB) {
  pdl_wait();
  pdl_trigger();
  const int cg = (C1 + C2) >> 3, cg1 = C1 >> 3;
  const int64_t total = M * cg;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int64_t m = idx / cg;
    const int c8 = (int)(idx % cg);
    if (!split) {
      const uint4 v = c8 < cg1 ? ldg16(A + m * C1 + c8 * 8) : ldg16(B + m * C2 + (c8 - cg1) * 8);
      stg16(OUT + m * (C1 + C2) + c8 * 8, v);
    } else {
      const uint4 v = ldg16(OUT + m * (C1 + C2) + c8 * 8);
      if (c8 < cg1) stg16(DA + m * C1 + c8 * 8, v);
      else stg16(DB + m * C2 + (c8 - cg1) * 8, v);
    }
  }
}

int cgrid(int64_t items) {
  int64_t g = (items + CNT - 1) / CNT;
  const int64_t cap = 16 * (int64_t)cvb_num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

extern "C" int cvb_im2col(const void* X, int x_fp32, int64_t sxn, int64_t sxc, int64_t sxh, int64_t sxw, int B, int Cin, int H, int W, int k, int stride,
                          int pad, void* A, int lda, cvb_stream_t stream) {
  CVB_CHECK(X && A && B > 0 && Cin > 0 && H > 0 && W > 0 && k > 0 && stride > 0 && pad >= 0, "cvb_im2col: bad arguments");
  CVB_CHECK(lda % 8 == 0 && lda >= k * k * Cin && cvb_aligned16(A), "cvb_im2col: lda must be a multiple of 8 and >= k*k*Cin");
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  CVB_CHECK(Ho > 0 && Wo > 0, "cvb_im2col: empty output");
  const int64_t M = (int64_t)B * Ho * Wo;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool nhwc = !x_fp32 && sxc == 1 && Cin % 8 == 0 && sxw == Cin && sxh == (int64_t)W * Cin && sxn == (int64_t)H * W * Cin && cvb_aligned16(X) &&
                    lda == k * k * Cin;
  if (nhwc) {
    CVB_CUDA(cvb_launch(im2col_nhwc_kernel, cgrid(M * k * k * (Cin / 8)), CNT, 0, st, static_cast<const bf16*>(X), Cin, H, W, k, stride, pad, Ho, Wo,
                        static_cast<bf16*>(A), lda, M));
  } else {
    CVB_CUDA(cvb_launch(im2col_generic_kernel, cgrid(M * lda), CNT, 0, st, X, x_fp32, sxn, sxc, sxh, sxw, Cin, H, W, k, stride, pad, Ho, Wo,
                        static_cast<bf16*>(A), lda, M));
  }
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_col2im(const void* dA, int lda, int B, int Cin, int H, int W, int k, int stride, int pad, void* dX, cvb_stream_t stream) {
  CVB_CHECK(dA && dX && B > 0 && Cin > 0 && Cin % 8 == 0 && H > 0 && W > 0 && k > 0 && stride > 0 && pad >= 0, "cvb_col2im: bad arguments (Cin %% 8 == 0)");
  CVB_CHECK(lda % 8 == 0 && lda >= k * k * Cin && cvb_aligned16(dA) && cvb_aligned16(dX), "cvb_col2im: bad leading dimension / alignment");
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const int64_t npix = (int64_t)B * H * W;
  CVB_CUDA(cvb_launch(col2im_nhwc_kernel, cgrid(npix * (Cin / 8)), CNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(dA), lda, Cin, H, W, k,
                      stride, pad, Ho, Wo, static_cast<bf16*>(dX), npix));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_patch_permute(const void* X, void* OUT, int B, int H, int W, int C, int patch_h, int patch_w, int inverse, cvb_stream_t stream) {
  CVB_CHECK(X && OUT && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && patch_h > 0 && patch_w > 0 && H % patch_h == 0 && W % patch_w == 0,
            "cvb_patch_permute: bad arguments (C %% 8 == 0, H, W multiples of the patch)");
  CVB_CHECK(cvb_aligned16(X) && cvb_aligned16(OUT), "cvb_patch_permute: misaligned operand");
  const int64_t npix = (int64_t)B * H * W;
  CVB_CUDA(cvb_launch(patch_permute_kernel, cgrid(npix * (C / 8)), CNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(X),
                      static_cast<bf16*>(OUT), H, W, C, patch_h, patch_w, inverse, npix));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_concat2(const void* A, const void* B, int C1, int C2, int64_t M, void* OUT, cvb_stream_t stream) {
  CVB_CHECK(A && B && OUT && C1 > 0 && C2 > 0 && C1 % 8 == 0 && C2 % 8 == 0 && M > 0, "cvb_concat2: bad arguments");
  CVB_CUDA(cvb_launch(concat2_kernel, cgrid(M * ((C1 + C2) / 8)), CNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(A),
                      static_cast<const bf16*>(B), static_cast<bf16*>(OUT), C1, C2, 0, M, static_cast<bf16*>(nullptr), static_cast<bf16*>(nullptr)));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_split2(const void* G, int C1, int C2, int64_t M, void* DA, void* DB, cvb_stream_t stream) {
  CVB_CHECK(G && DA && DB && C1 > 0 && C2 > 0 && C1 % 8 == 0 && C2 % 8 == 0 && M > 0, "cvb_split2: bad arguments");
  CVB_CUDA(cvb_launch(concat2_kernel, cgrid(M * ((C1 + C2) / 8)), CNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(nullptr),
                      static_cast<const bf16*>(nullptr), const_cast<bf16*>(static_cast<const bf16*>(G)), C1, C2, 1, M, static_cast<bf16*>(DA),
                      static_cast<bf16*>(DB)));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_vit_tokens_interp_fwd(const void* patch, const float* pos, int n_pos, const float* cls, void* out, int B, int N, int C,
                                         cvb_stream_t stream) {
  CVB_CHECK(patch && pos && out && B > 0 && N > 0 && n_pos > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(patch) && cvb_aligned16(out),
            "cvb_vit_tokens_interp_fwd: bad arguments");
  const int has_cls = cls != nullptr;
  CVB_CUDA(cvb_launch(vit_tokens_interp_fwd_kernel, cgrid((int64_t)B * (N + has_cls) * (C / 8)), CNT, 0, static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(patch), pos, n_pos, (float)n_pos / (float)N, cls, static_cast<bf16*>(out), B, N, C, has_cls));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_vit_tokens_interp_bwd(const void* dout, void* dpatch, float* dpos, int n_pos, float* dcls, int B, int N, int C, cvb_stream_t stream) {
  CVB_CHECK(dout && dpatch && dpos && B > 0 && N > 0 && n_pos > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(dout) && cvb_aligned16(dpatch),
            "cvb_vit_tokens_interp_bwd: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int has_cls = dcls != nullptr;
  // batch sum per output token into a zeroed fp32 [N, C] scratch (vit_tokens_bwd_kernel, dpos = scratch), then the transposed stencil
  double* ws = nullptr;
  if (cvb_det_alloc(&ws, ((size_t)N * C + 1) / 2, st)) return 2;
  float* g = reinterpret_cast<float*>(ws);
  CVB_CUDA(cvb_launch(vit_tokens_bwd_kernel, cgrid((int64_t)(N + has_cls) * (C / 8)), CNT, 0, st, static_cast<const bf16*>(dout), static_cast<bf16*>(dpatch),
                      g, dcls, B, N, C, has_cls));
  CVB_LAUNCH_CHECK();
  CVB_CUDA(cvb_launch(vit_pos_interp_bwd_kernel, cgrid((int64_t)n_pos * (C / 8)), CNT, 0, st, static_cast<const float*>(g), dpos, n_pos,
                      (float)n_pos / (float)N, N, C));
  CVB_LAUNCH_CHECK();
  return cvb_det_free(ws, st);
}
