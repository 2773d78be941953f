// CLIP text tower edges and feature normalisation (BASELINE.json configs[4]; SURVEY.md 8f row 2), sm_90a.
//   cvb_embedding_{fwd,bwd} : token embedding + learnable positional embedding (cvnets/text_encoders/transformer.py:328-341,
//                             cvnets/layers/embedding.py, positional_embedding.py:53-110)
//   cvb_eot_gather_{fwd,bwd}: features of the end-of-text token = the highest token id of each sequence (transformer.py:413-421)
//   cvb_l2norm_{fwd,bwd}    : F.normalize(x, dim=-1) of the projected image / text features (transformer.py:423-425,
//                             image_projection_layers/simple_projection_head.py)
// Everything else of the CLIP step reuses the library: TransformerEncoder (causal additive mask), the ViT image tower, the projection
// matmuls (cvb_pw_gemm / cvb_pw_wgrad), the two cross-entropies of the contrastive loss (cvb_ce_* with the logit scale folded in).
#include "common.cuh"

namespace {

constexpr int KNT = 256;

__global__ void __launch_bounds__(KNT) embedding_fwd_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ table, const float* __restrict__ pos,
                                                            bf16* __restrict__ out, int64_t ntok, int S, int C, int V) {
  pdl_wait();
  pdl_trigger();
  const int cg = C >> 3;
  const int64_t total = ntok * cg;
  for (int64_t idx = (int64_t)blockIdx.x * KNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * KNT) {
    const int64_t t = idx / cg;
    const int c8 = (int)(idx % cg);
    int64_t id = tokens[t];
    if (id < 0 || id >= V) id = 0;
    const float* src = table + id * C + c8 * 8;
    float f[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) f[q] = src[q];
    if (pos) {
      const float* ps = pos + (int64_t)(t % S) * C + c8 * 8;
#pragma unroll
      for (int q = 0; q < 8; ++q) f[q] += ps[q];
    }
    stg16(out + t * C + c8 * 8, pack8(f));
  }
}

// dtable[token] += dout (fp32 atomics: a vocabulary row may be hit by many tokens); dpos[s] += sum_b dout[b, s]
__global__ void __launch_bounds__(KNT) embedding_bwd_kernel(const bf16* __restrict__ dout, const int64_t* __restrict__ tokens, float* __restrict__ dtable,
                                                            float* __restrict__ dpos, int64_t ntok, int S, int C, int V) {
  pdl_wait();
  pdl_trigger();
  const int cg = C >> 3;
  const int64_t total = ntok * cg;
  for (int64_t idx = (int64_t)blockIdx.x * KNT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * KNT) {
    const int64_t t = idx / cg;
    const int c8 = (int)(idx % cg);
    float f[8];
    unpack8(ldg16(dout + t * C + c8 * 8), f);
    const int64_t id = tokens[t];
    if (id >= 0 && id < V) {
      float* dst = dtable + id * C + c8 * 8;
#pragma unroll
      for (int q = 0; q < 8; ++q) atomicAdd(dst + q, f[q]);
    }
    if (dpos) {
      float* dp = dpos + (int64_t)(t % S) * C + c8 * 8;
#pragma unroll
      for (int q = 0; q < 8; ++q) atomicAdd(dp + q, f[q]);
    }
  }
}

// one CTA per sequence: argmax of the token ids (first maximum, like torch.argmax), then copy that token's row
__global__ void __launch_bounds__(128) eot_gather_fwd_kernel(const bf16* __restrict__ X, const int64_t* __restrict__ tokens, int S, int C,
                                                             bf16* __restrict__ out, int* __restrict__ idx_out) {
  pdl_wait();
  pdl_trigger();
  __shared__ int s_idx;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int best = 0;
    int64_t bv = tokens[(int64_t)b * S];
    for (int s = 1; s < S; ++s) {
      const int64_t v = tokens[(int64_t)b * S + s];
      if (v > bv) { bv = v; best = s; }
    }
    s_idx = best;
    idx_out[b] = best;
  }
  __syncthreads();
  const bf16* src = X + ((int64_t)b * S + s_idx) * C;
  for (int c = threadIdx.x * 8; c < C; c += blockDim.x * 8) stg16(out + (int64_t)b * C + c, ldg16(src + c));
}

// dX = 0 everywhere except the gathered rows
__global__ void __launch_bounds__(KNT) eot_gather_bwd_kernel(const bf16* __restrict__ dout, const int* __restrict__ idx, int S, int C, bf16* __restrict__ dX,
                                                             int64_t ntok) {
  pdl_wait();
  pdl_trigger();
  const int cg = C >> 3;
  const int64_t total = ntok * cg;
  for (int64_t i = (int64_t)blockIdx.x * KNT + threadIdx.x; i < total; i += (int64_t)gridDim.x * KNT) {
    const int64_t t = i / cg;
    const int c8 = (int)(i % cg);
    const int64_t b = t / S;
    const int s = (int)(t % S);
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (s == idx[b]) v = ldg16(dout + b * C + c8 * 8);
    stg16(dX + t * C + c8 * 8, v);
  }
}

// y = x / max(||x||, eps): one warp per row
__global__ void __launch_bounds__(KNT) l2norm_fwd_kernel(const bf16* __restrict__ X, bf16* __restrict__ Y, float* __restrict__ inv_norm, int M, int C,
                                                         float eps) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (KNT / 32) + (threadIdx.x >> 5);
  if (row >= M) return;
  const bf16* x = X + (int64_t)row * C;
  float q = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    float f[8];
    unpack8(ldg16(x + c), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) q = fmaf(f[e], f[e], q);
  }
  q = warp_sum(q);
  const float inv = 1.0f / fmaxf(sqrtf(q), eps);
  if (lane == 0) inv_norm[row] = inv;
  for (int c = lane * 8; c < C; c += 256) {
    float f[8];
    unpack8(ldg16(x + c), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] *= inv;
    stg16(Y + (int64_t)row * C + c, pack8(f));
  }
}

// dx = inv * (dy - y * (y . dy))   (rows whose norm was clamped by eps are degenerate and treated like the generic case)
__global__ void __launch_bounds__(KNT) l2norm_bwd_kernel(const bf16* __restrict__ DY, const bf16* __restrict__ Y, const float* __restrict__ inv_norm,
                                                         bf16* __restrict__ DX, int M, int C) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (KNT / 32) + (threadIdx.x >> 5);
  if (row >= M) return;
  const bf16* dy = DY + (int64_t)row * C;
  const bf16* y = Y + (int64_t)row * C;
  float dot = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    float a[8], b[8];
    unpack8(ldg16(dy + c), a);
    unpack8(ldg16(y + c), b);
#pragma unroll
    for (int e = 0; e < 8; ++e) dot = fmaf(a[e], b[e], dot);
  }
  dot = warp_sum(dot);
  const float inv = inv_norm[row];
  for (int c = lane * 8; c < C; c += 256) {
    float a[8], b[8];
    unpack8(ldg16(dy + c), a);
    unpack8(ldg16(y + c), b);
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] = inv * (a[e] - b[e] * dot);
    stg16(DX + (int64_t)row * C + c, pack8(a));
  }
}

int kgrid(int64_t items) {
  int64_t g = (items + KNT - 1) / KNT;
  const int64_t cap = 16 * (int64_t)cvb_num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

extern "C" int cvb_embedding_fwd(const int64_t* tokens, const float* table, const float* pos, void* out, int B, int S, int C, int V, cvb_stream_t stream) {
  CVB_CHECK(tokens && table && out && B > 0 && S > 0 && C > 0 && C % 8 == 0 && V > 0 && cvb_aligned16(out), "cvb_embedding_fwd: bad arguments");
  const int64_t ntok = (int64_t)B * S;
  CVB_CUDA(cvb_launch(embedding_fwd_kernel, kgrid(ntok * (C / 8)), KNT, 0, static_cast<cudaStream_t>(stream), tokens, table, pos, static_cast<bf16*>(out), ntok,
                      S, C, V));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_embedding_bwd(const void* dout, const int64_t* tokens, float* dtable, float* dpos, int B, int S, int C, int V, cvb_stream_t stream) {
  CVB_CHECK(dout && tokens && dtable && B > 0 && S > 0 && C > 0 && C % 8 == 0 && V > 0 && cvb_aligned16(dout), "cvb_embedding_bwd: bad arguments");
  const int64_t ntok = (int64_t)B * S;
  CVB_CUDA(cvb_launch(embedding_bwd_kernel, kgrid(ntok * (C / 8)), KNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(dout), tokens, dtable,
                      dpos, ntok, S, C, V));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_eot_gather_fwd(const void* X, const int64_t* tokens, int B, int S, int C, void* out, int* idx, cvb_stream_t stream) {
  CVB_CHECK(X && tokens && out && idx && B > 0 && S > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(X) && cvb_aligned16(out), "cvb_eot_gather_fwd: bad arguments");
  CVB_CUDA(cvb_launch(eot_gather_fwd_kernel, B, 128, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(X), tokens, S, C, static_cast<bf16*>(out),
                      idx));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_eot_gather_bwd(const void* dout, const int* idx, int B, int S, int C, void* dX, cvb_stream_t stream) {
  CVB_CHECK(dout && idx && dX && B > 0 && S > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(dout) && cvb_aligned16(dX), "cvb_eot_gather_bwd: bad arguments");
  const int64_t ntok = (int64_t)B * S;
  CVB_CUDA(cvb_launch(eot_gather_bwd_kernel, kgrid(ntok * (C / 8)), KNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(dout), idx, S, C,
                      static_cast<bf16*>(dX), ntok));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_l2norm_fwd(const void* X, void* Y, float* inv_norm, int M, int C, float eps, cvb_stream_t stream) {
  CVB_CHECK(X && Y && inv_norm && M > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(X) && cvb_aligned16(Y), "cvb_l2norm_fwd: bad arguments");
  CVB_CUDA(cvb_launch(l2norm_fwd_kernel, (M + KNT / 32 - 1) / (KNT / 32), KNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(X),
                      static_cast<bf16*>(Y), inv_norm, M, C, eps));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_l2norm_bwd(const void* DY, const void* Y, const float* inv_norm, void* DX, int M, int C, cvb_stream_t stream) {
  CVB_CHECK(DY && Y && inv_norm && DX && M > 0 && C > 0 && C % 8 == 0 && cvb_aligned16(DY) && cvb_aligned16(Y) && cvb_aligned16(DX), "cvb_l2norm_bwd: bad arguments");
  CVB_CUDA(cvb_launch(l2norm_bwd_kernel, (M + KNT / 32 - 1) / (KNT / 32), KNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(DY),
                      static_cast<const bf16*>(Y), inv_norm, static_cast<bf16*>(DX), M, C));
  CVB_LAUNCH_CHECK();
  return 0;
}
