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

// MobileViT-v1 unfolding / folding of a map that is not a multiple of the patch (mobilevit_block.py:191-200, :259-265): the reference resizes
// the H x W map bilinearly (align_corners=False) up to the Hn x Wn grid the patches tile before unfolding, and the folded Hn x Wn map back down
// to H x W.  Each kernel thread owns one output row (8 channels) and fuses the resample with the row permutation; row indices on the Hn x Wn
// grid are token rows (b*P + p, n).  interp_src is PyTorch's source-index rule per axis, scale = n_src / n_dst.
//   dir 0 (unfold)  token (y, x) of Hn x Wn = the 4-tap stencil of map H x W             dir 2 = transpose of 0: map pixel (y, x) gathers
//   dir 1 (fold)    map pixel (y, x) of H x W = the 4-tap stencil of the token grid        the tokens whose dir-0 stencil reads it
//                                                                                          dir 3 = transpose of 1: token (y, x) gathers the map
// Transposes are gathers over the few destinations whose stencil touches the row (like vit_pos_interp_bwd_kernel): no atomics, the same
// bits every run.  fp32 arithmetic, one bf16 rounding.
__device__ __forceinline__ int64_t grid_row(int64_t b, int y, int x, int Hg, int Wg, bool tok, int ph, int pw) {
  if (!tok) return (b * Hg + y) * Wg + x;
  const int nw = Wg / pw, N = (Hg / ph) * nw;
  return (b * (ph * pw) + (y % ph) * pw + (x % pw)) * N + (y / ph) * nw + (x / pw);
}
// the weight with which destination d of a 1-D stencil (n_src sources, scale) reads source j; false if it does not read it
__device__ __forceinline__ bool stencil_weight(int d, int j, float scale, int n_src, float& w) {
  int i0, i1;
  float lam;
  interp_src(d, scale, n_src, i0, i1, lam);
  if (i0 != j && i1 != j) return false;
  w = i0 == j ? __fsub_rn(1.f, lam) : 0.f;
  if (i1 == j) w = __fadd_rn(w, lam);
  return true;
}
__global__ void __launch_bounds__(CNT) patch_resample_kernel(const bf16* __restrict__ X, bf16* __restrict__ OUT, int H, int W, int Hn, int Wn, int C,
                                                             int ph, int pw, int dir, int64_t nrows) {
  pdl_wait();
  pdl_trigger();
  // the stencil runs from its source grid (sh x sw) to its destination grid (dh x dw): map -> tokens for dirs 0 / 2, tokens -> map for 1 / 3
  const bool up = dir == 0 || dir == 2, adjoint = dir >= 2;
  const int sh = up ? H : Hn, sw = up ? W : Wn, dh = up ? Hn : H, dw = up ? Wn : W;
  const float sy = (float)sh / (float)dh, sx = (float)sw / (float)dw;
  // a forward direction writes the destination grid and reads the source grid; its transpose the other way round
  const int oh = adjoint ? sh : dh, ow = adjoint ? sw : dw, ih = adjoint ? dh : sh, iw = adjoint ? dw : sw;
  const bool out_tok = (dir == 0 || dir == 3), in_tok = !out_tok;
  const int cg = C >> 3;
  const int64_t total = nrows * cg;
  for (int64_t idx = (int64_t)blockIdx.x * CNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * CNT) {
    const int64_t pix = idx / cg;
    const int c8 = (int)(idx % cg);
    const int x = (int)(pix % ow), y = (int)((pix / ow) % oh);
    const int64_t b = pix / ((int64_t)ow * oh);
    float acc[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] = 0.f;
    if (!adjoint) {
      int y0, y1, x0, x1;
      float ly, lx;
      interp_src(y, sy, sh, y0, y1, ly);
      interp_src(x, sx, sw, x0, x1, lx);
      const int ys[2] = {y0, y1}, xs[2] = {x0, x1};
      const float wy[2] = {__fsub_rn(1.f, ly), ly}, wx[2] = {__fsub_rn(1.f, lx), lx};
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        float row[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) row[q] = 0.f;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float f[8];
          unpack8(ldg16(X + grid_row(b, ys[a], xs[e], ih, iw, in_tok, ph, pw) * C + c8 * 8), f);
#pragma unroll
          for (int q = 0; q < 8; ++q) row[q] = __fadd_rn(row[q], __fmul_rn(wx[e], f[q]));
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = __fadd_rn(acc[q], __fmul_rn(wy[a], row[q]));
      }
    } else {
      // destinations whose source index i0 lies in {j - 1, j}: src in [j - 1, j + 1), widened by 2 (vit_pos_interp_bwd_kernel)
      const int d_lo = max(0, (int)((y - 1.0f) / sy) - 2), d_hi = min(dh - 1, (int)((y + 2.0f) / sy) + 2);
      const int e_lo = max(0, (int)((x - 1.0f) / sx) - 2), e_hi = min(dw - 1, (int)((x + 2.0f) / sx) + 2);
      for (int d = d_lo; d <= d_hi; ++d) {
        float wy;
        if (!stencil_weight(d, y, sy, sh, wy)) continue;
        float row[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) row[q] = 0.f;
        for (int e = e_lo; e <= e_hi; ++e) {
          float wx;
          if (!stencil_weight(e, x, sx, sw, wx)) continue;
          float f[8];
          unpack8(ldg16(X + grid_row(b, d, e, ih, iw, in_tok, ph, pw) * C + c8 * 8), f);
#pragma unroll
          for (int q = 0; q < 8; ++q) row[q] = __fadd_rn(row[q], __fmul_rn(wx, f[q]));
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = __fadd_rn(acc[q], __fmul_rn(wy, row[q]));
      }
    }
    stg16(OUT + grid_row(b, y, x, oh, ow, out_tok, ph, pw) * C + c8 * 8, pack8(acc));
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
  return 0;
}

extern "C" int cvb_col2im(const void* dA, int lda, int B, int Cin, int H, int W, int k, int stride, int pad, void* dX, cvb_stream_t stream) {
  CVB_CHECK(dA && dX && B > 0 && Cin > 0 && Cin % 8 == 0 && H > 0 && W > 0 && k > 0 && stride > 0 && pad >= 0, "cvb_col2im: bad arguments (Cin %% 8 == 0)");
  CVB_CHECK(lda % 8 == 0 && lda >= k * k * Cin && cvb_aligned16(dA) && cvb_aligned16(dX), "cvb_col2im: bad leading dimension / alignment");
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  const int64_t npix = (int64_t)B * H * W;
  CVB_CUDA(cvb_launch(col2im_nhwc_kernel, cgrid(npix * (Cin / 8)), CNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(dA), lda, Cin, H, W, k,
                      stride, pad, Ho, Wo, static_cast<bf16*>(dX), npix));
  return 0;
}

extern "C" int cvb_patch_permute(const void* X, void* OUT, int B, int H, int W, int C, int patch_h, int patch_w, int direction,
                                 cvb_stream_t stream) {
  CVB_CHECK(X && OUT && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && patch_h > 0 && patch_w > 0, "cvb_patch_permute: bad arguments (C %% 8 == 0)");
  CVB_CHECK(direction >= CVB_PATCH_UNFOLD && direction <= CVB_PATCH_FOLD_T, "cvb_patch_permute: direction %d is not a cvb_patch_direction", direction);
  CVB_CHECK(cvb_aligned16(X) && cvb_aligned16(OUT), "cvb_patch_permute: misaligned operand");
  const int Hn = (H + patch_h - 1) / patch_h * patch_h, Wn = (W + patch_w - 1) / patch_w * patch_w;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (Hn == H && Wn == W) {  // a row permutation, its own adjoint with the direction flipped
    const int64_t npix = (int64_t)B * H * W;
    const int inverse = direction == CVB_PATCH_FOLD || direction == CVB_PATCH_UNFOLD_T;
    CVB_CUDA(cvb_launch(patch_permute_kernel, cgrid(npix * (C / 8)), CNT, 0, st, static_cast<const bf16*>(X), static_cast<bf16*>(OUT), H, W, C, patch_h,
                        patch_w, inverse, npix));
    return 0;
  }
  const bool tok_out = direction == CVB_PATCH_UNFOLD || direction == CVB_PATCH_FOLD_T;
  const int64_t nrows = (int64_t)B * (tok_out ? (int64_t)Hn * Wn : (int64_t)H * W);
  CVB_CUDA(cvb_launch(patch_resample_kernel, cgrid(nrows * (C / 8)), CNT, 0, st, static_cast<const bf16*>(X), static_cast<bf16*>(OUT), H, W, Hn, Wn, C,
                      patch_h, patch_w, direction, nrows));
  return 0;
}

extern "C" int cvb_concat2(const void* A, const void* B, int C1, int C2, int64_t M, void* OUT, cvb_stream_t stream) {
  CVB_CHECK(A && B && OUT && C1 > 0 && C2 > 0 && C1 % 8 == 0 && C2 % 8 == 0 && M > 0, "cvb_concat2: bad arguments");
  CVB_CUDA(cvb_launch(concat2_kernel, cgrid(M * ((C1 + C2) / 8)), CNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(A),
                      static_cast<const bf16*>(B), static_cast<bf16*>(OUT), C1, C2, 0, M, static_cast<bf16*>(nullptr), static_cast<bf16*>(nullptr)));
  return 0;
}

extern "C" int cvb_split2(const void* G, int C1, int C2, int64_t M, void* DA, void* DB, cvb_stream_t stream) {
  CVB_CHECK(G && DA && DB && C1 > 0 && C2 > 0 && C1 % 8 == 0 && C2 % 8 == 0 && M > 0, "cvb_split2: bad arguments");
  CVB_CUDA(cvb_launch(concat2_kernel, cgrid(M * ((C1 + C2) / 8)), CNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(nullptr),
                      static_cast<const bf16*>(nullptr), const_cast<bf16*>(static_cast<const bf16*>(G)), C1, C2, 1, M, static_cast<bf16*>(DA),
                      static_cast<bf16*>(DB)));
  return 0;
}

extern "C" int cvb_vit_tokens_interp_fwd(const void* patch, const float* pos, int n_pos, const float* cls, void* out, int B, int N, int C,
                                         cvb_stream_t stream) {
  CVB_CHECK(patch && pos && out && B > 0 && N > 0 && n_pos > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(patch) && cvb_aligned16(out),
            "cvb_vit_tokens_interp_fwd: bad arguments");
  const int has_cls = cls != nullptr;
  CVB_CUDA(cvb_launch(vit_tokens_interp_fwd_kernel, cgrid((int64_t)B * (N + has_cls) * (C / 8)), CNT, 0, static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(patch), pos, n_pos, (float)n_pos / (float)N, cls, static_cast<bf16*>(out), B, N, C, has_cls));
  return 0;
}

extern "C" int cvb_vit_tokens_interp_bwd(const void* dout, void* dpatch, float* dpos, int n_pos, float* dcls, int B, int N, int C, cvb_stream_t stream) {
  CVB_CHECK(dout && dpatch && dpos && B > 0 && N > 0 && n_pos > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(dout) && cvb_aligned16(dpatch),
            "cvb_vit_tokens_interp_bwd: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int has_cls = dcls != nullptr;
  // batch sum per output token into a zeroed fp32 [N, C] scratch (vit_tokens_bwd_kernel, dpos = scratch), then the transposed stencil
  DetScratch ws(st);
  if (ws.alloc(((size_t)N * C + 1) / 2)) return 2;
  float* g = reinterpret_cast<float*>(ws.data());
  CVB_CUDA(cvb_launch(vit_tokens_bwd_kernel, cgrid((int64_t)(N + has_cls) * (C / 8)), CNT, 0, st, static_cast<const bf16*>(dout), static_cast<bf16*>(dpatch),
                      g, dcls, B, N, C, has_cls));
  CVB_CUDA(cvb_launch(vit_pos_interp_bwd_kernel, cgrid((int64_t)n_pos * (C / 8)), CNT, 0, st, static_cast<const float*>(g), dpos, n_pos,
                      (float)n_pos / (float)N, N, C));
  return ws.release();
}
