// LinearSelfAttention core (MobileViTv2) between qkv_proj and out_proj, forward and backward (sm_90a).
// Reference: cvnets/layers/linear_attention.py:134-161; math: SURVEY.md Appendix A5.
//
// unfold / fold (cvnets/modules/mobilevit_block.py:526-555) never materialise: the tensor stays the channels-last feature
// map [B, H, W, ld]; "pixel position p of patch n" is pixel (2*(n / (W/2)) + p/2, 2*(n % (W/2)) + p%2).  One CTA owns one
// (sample, p) pair: softmax over its N patches, the context reduction over N and the broadcast product all stay on chip;
// qkv is read once and the output written once (O(B*d*P*N), no N x N matrix exists in this attention).
#include "common.cuh"

namespace {

constexpr int NT = 256;

// unf != 0: the tensor is the UNFOLDED [B, P, N, ld] matrix itself (stand-alone LinearSelfAttention on a [B, d, P, N] input,
// linear_attention.py:134-207): H = P, W = N and row (b, p, n) is the plain row-major index.
__device__ __forceinline__ int64_t pix_index(int b, int p, int n, int H, int W, int unf = 0) {
  if (unf) return ((int64_t)b * H + p) * W + n;
  const int nw = W >> 1;
  const int h = 2 * (n / nw) + (p >> 1), w = 2 * (n % nw) + (p & 1);
  return ((int64_t)b * H + h) * W + w;
}

__device__ float block_reduce_sum(float v, float* ws) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < (int)(blockDim.x + 31) / 32; ++i) t += ws[i];
  return t;
}
__device__ float block_reduce_max(float v, float* ws) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
  for (int i = 0; i < (int)(blockDim.x + 31) / 32; ++i) t = fmaxf(t, ws[i]);
  return t;
}

// Rows whose 16-byte loads a thread issues together.  Every loop over a thread's rows n = grp, grp + ngrp, ... keeps that ascending order, so
// the fp32 chains it accumulates do not depend on the batching; the first batch of each pass is loaded before the barrier that precedes it.
constexpr int LA_U = 4;

__device__ __forceinline__ void load_rows(uint4 (&v)[LA_U], const bf16* base, int ld, int col, int b, int p, int n0, int step, int N, int H, int W,
                                          int unf) {
#pragma unroll
  for (int u = 0; u < LA_U; ++u) {
    const int n = n0 + u * step;
    if (n < N) v[u] = ldg16(base + pix_index(b, p, n, H, W, unf) * ld + col);
  }
}

// dynamic smem: s[N] | ctx[d] | partials[ngrp][d]
// Cross-attention (linear_attention.py:163-207): query/key come from QKV (N rows per (b, p), the "previous" tensor), the values and the
// output live in VX / O with Nv rows per (b, p); self-attention passes VX = QKV, Nv = N.
__global__ void __launch_bounds__(NT) linattn_fwd_kernel(const bf16* __restrict__ QKV, int ldq, int H, int W, int d, bf16* __restrict__ O, int ldo,
                                                         float* __restrict__ S, float* __restrict__ CTX, int unf, const bf16* __restrict__ VX,
                                                         int ldvx, int Nv) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];
  __shared__ float ws[NT / 32];
  const int N = unf ? W : (H >> 1) * (W >> 1);
  const int P = unf ? H : 4;
  const int Wv = (VX == QKV) ? W : Nv;  // cross-attention is unfolded-only: row (b, p, n) of a [B, P, Nv, *] matrix
  float* s_s = sm;
  float* s_ctx = sm + N;
  const int b = blockIdx.x / P, p = blockIdx.x % P;
  const int tid = threadIdx.x;
  const int cgs = d >> 3;
  const int cg = tid % cgs, grp = tid / cgs, ngrp = blockDim.x / cgs;
  const int n_first = grp < ngrp ? grp : N;  // threads beyond cgs*ngrp only take part in the block-wide steps
  const int nv_first = grp < ngrp ? grp : Nv;
  uint4 kb[LA_U];
  load_rows(kb, QKV, ldq, cg * 8, b, p, n_first, ngrp, N, H, W, unf);

  // softmax over the N patches of the query channel (column 2d)
  float lmax = -INFINITY;
  for (int n = tid; n < N; n += blockDim.x) {
    float q = __bfloat162float(QKV[pix_index(b, p, n, H, W, unf) * ldq + 2 * d]);
    s_s[n] = q;
    lmax = fmaxf(lmax, q);
  }
  const float gmax = block_reduce_max(lmax, ws);
  float lsum = 0.f;
  for (int n = tid; n < N; n += blockDim.x) {
    float e = __expf(s_s[n] - gmax);
    s_s[n] = e;
    lsum += e;
  }
  const float inv = 1.f / block_reduce_sum(lsum, ws);
  for (int n = tid; n < N; n += blockDim.x) {
    float sv = s_s[n] * inv;
    s_s[n] = sv;
    S[((int64_t)b * P + p) * N + n] = sv;
  }
  __syncthreads();

  // ctx[c] = sum_n key[n,c] * s[n]
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int n0 = n_first; n0 < N; n0 += LA_U * ngrp) {
    if (n0 != n_first) load_rows(kb, QKV, ldq, cg * 8, b, p, n0, ngrp, N, H, W, unf);
#pragma unroll
    for (int u = 0; u < LA_U; ++u) {
      const int n = n0 + u * ngrp;
      if (n >= N) break;
      float k[8];
      unpack8(kb[u], k);
      const float sv = s_s[n];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(k[j], sv, acc[j]);
    }
  }
  uint4 vb[LA_U];
  load_rows(vb, VX, ldvx, d + cg * 8, b, p, nv_first, ngrp, Nv, H, Wv, unf);
  // deterministic cross-group reduction (fixed order): partials -> smem [ngrp][d] -> ordered sum
  float* s_part = s_ctx + d;
  if (grp < ngrp) {
#pragma unroll
    for (int j = 0; j < 8; ++j) s_part[grp * d + cg * 8 + j] = acc[j];
  }
  __syncthreads();
  for (int i = tid; i < d; i += blockDim.x) {
    float t = 0.f;
    for (int gq = 0; gq < ngrp; ++gq) t += s_part[gq * d + i];
    s_ctx[i] = t;
    CTX[((int64_t)b * P + p) * d + i] = t;
  }
  __syncthreads();
  float ctx[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) ctx[j] = s_ctx[cg * 8 + j];
  // O = relu(value) * ctx
  for (int n0 = nv_first; n0 < Nv; n0 += LA_U * ngrp) {
    if (n0 != nv_first) load_rows(vb, VX, ldvx, d + cg * 8, b, p, n0, ngrp, Nv, H, Wv, unf);
#pragma unroll
    for (int u = 0; u < LA_U; ++u) {
      const int n = n0 + u * ngrp;
      if (n >= Nv) break;
      float v[8];
      unpack8(vb[u], v);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f) * ctx[j];
      stg16(O + pix_index(b, p, n, H, Wv, unf) * ldo + cg * 8, pack8(v));
    }
  }
}

// The channel groups of one row n are the cgs consecutive threads grp * cgs .. grp * cgs + cgs - 1; they span at most la_pieces(cgs) warps.
__host__ __device__ inline int la_pieces(int cgs) {
  int q = 1;
  for (int g = 0; g < NT / cgs; ++g) {
    const int w = (g * cgs + cgs - 1) / 32 - (g * cgs) / 32 + 1;
    q = w > q ? w : q;
  }
  return q;
}

// dynamic smem: dsp[npc][N] | dctx[d] | dbk[d] | dbv[d] (fp64) | part[2][ngrp][d] | s[N] | ctx[d] (fp32)
// Every sum that several threads contribute to is fp64 and fixed-order: the warp pieces of a row's ds by shuffles, the cross-group partials of
// dctx, dbv and dbk through part[].
__global__ void __launch_bounds__(NT) linattn_bwd_kernel(const bf16* __restrict__ QKV, int ldq, const bf16* __restrict__ DO, int ldo,
                                                         const float* __restrict__ S, const float* __restrict__ CTX, int H, int W, int d,
                                                         bf16* __restrict__ DQKV, double* __restrict__ dbias, int unf, const bf16* __restrict__ VX,
                                                         int ldvx, int Nv, bf16* __restrict__ DVX) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ double smd[];
  __shared__ float ws[NT / 32];
  const int N = unf ? W : (H >> 1) * (W >> 1);
  const int P = unf ? H : 4;
  const int Wv = (VX == QKV) ? W : Nv;
  const int cgs = d >> 3;
  const int npc = la_pieces(cgs);
  const int ngrp = blockDim.x / cgs;
  double* s_dsp = smd;
  double* s_dctx = s_dsp + (size_t)npc * N;
  double* s_dbk = s_dctx + d;
  double* s_dbv = s_dbk + d;
  float* s_part = reinterpret_cast<float*>(s_dbv + d);
  float* s_s = s_part + 2 * ngrp * d;
  float* s_ctx = s_s + N;
  const int b = blockIdx.x / P, p = blockIdx.x % P;
  const int tid = threadIdx.x;
  const int cg = tid % cgs, grp = tid / cgs;
  const int n_first = grp < ngrp ? grp : N;
  const int nv_first = grp < ngrp ? grp : Nv;
  uint4 vb[LA_U], gb[LA_U];
  load_rows(vb, VX, ldvx, d + cg * 8, b, p, nv_first, ngrp, Nv, H, Wv, unf);
  load_rows(gb, DO, ldo, cg * 8, b, p, nv_first, ngrp, Nv, H, Wv, unf);
  for (int n = tid; n < N; n += blockDim.x) s_s[n] = S[((int64_t)b * P + p) * N + n];
  for (int i = tid; i < npc * N; i += blockDim.x) s_dsp[i] = 0.0;
  for (int i = tid; i < d; i += blockDim.x) s_ctx[i] = CTX[((int64_t)b * P + p) * d + i];
  __syncthreads();

  // pass 1: dctx[c] = sum_n dO*relu(V);  dV = dO * ctx * 1[V>0]
  {
    float ctx[8], acc[8], dbv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { ctx[j] = s_ctx[cg * 8 + j]; acc[j] = 0.f; dbv[j] = 0.f; }
    for (int n0 = nv_first; n0 < Nv; n0 += LA_U * ngrp) {
      if (n0 != nv_first) {
        load_rows(vb, VX, ldvx, d + cg * 8, b, p, n0, ngrp, Nv, H, Wv, unf);
        load_rows(gb, DO, ldo, cg * 8, b, p, n0, ngrp, Nv, H, Wv, unf);
      }
#pragma unroll
      for (int u = 0; u < LA_U; ++u) {
        const int n = n0 + u * ngrp;
        if (n >= Nv) break;
        float v[8], g[8];
        unpack8(vb[u], v);
        unpack8(gb[u], g);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool pos = v[j] > 0.f;
          acc[j] = fmaf(g[j], pos ? v[j] : 0.f, acc[j]);
          g[j] = pos ? bf16_round(g[j] * ctx[j]) : 0.f;
          dbv[j] += g[j];
        }
        stg16(DVX + pix_index(b, p, n, H, Wv, unf) * ldvx + d + cg * 8, pack8(g));
      }
    }
    if (grp < ngrp) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { s_part[grp * d + cg * 8 + j] = acc[j]; s_part[(ngrp + grp) * d + cg * 8 + j] = dbv[j]; }
    }
  }
  uint4 kb[LA_U];
  load_rows(kb, QKV, ldq, cg * 8, b, p, n_first, ngrp, N, H, W, unf);
  __syncthreads();
  for (int i = tid; i < d; i += blockDim.x) {
    double t = 0.0, tv = 0.0;
    for (int gq = 0; gq < ngrp; ++gq) { t += (double)s_part[gq * d + i]; tv += (double)s_part[(ngrp + gq) * d + i]; }
    s_dctx[i] = t;
    s_dbv[i] = tv;
  }
  __syncthreads();
  // pass 2: ds[n] = sum_c dctx[c]*K[n,c];  dK = dctx * s[n].  The trip count is the same for every thread (the row reductions are warp
  // shuffles); a thread's row n = grp + k * ngrp is real when grp < ngrp and n < N.
  {
    const int lane = tid & 31, warp = tid >> 5;
    // this thread's row occupies lanes [seg_lo, seg_hi] of the warp; threads without a row form one-lane segments
    const int seg_lo = grp < ngrp ? max(grp * cgs - warp * 32, 0) : lane;
    const int seg_hi = grp < ngrp ? min(grp * cgs + cgs - 1 - warp * 32, 31) : lane;
    const int piece = warp - (grp * cgs) / 32;
    float dctx[8], dbk[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { dctx[j] = (float)s_dctx[cg * 8 + j]; dbk[j] = 0.f; }
    const int steps = (N + ngrp - 1) / ngrp;
    for (int k0 = 0; k0 < steps; k0 += LA_U) {
      const int n0 = grp + k0 * ngrp;
      if (k0 != 0) load_rows(kb, QKV, ldq, cg * 8, b, p, grp < ngrp ? n0 : N, ngrp, N, H, W, unf);
#pragma unroll
      for (int u = 0; u < LA_U; ++u) {
        if (k0 + u >= steps) break;
        const int n = n0 + u * ngrp;
        const bool real = grp < ngrp && n < N;
        double part = 0.0;
        if (real) {
          float k[8], dk[8];
          unpack8(kb[u], k);
          const float sv = s_s[n];
          float pf = 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            pf = fmaf(dctx[j], k[j], pf);
            dk[j] = bf16_round(dctx[j] * sv);
            dbk[j] += dk[j];
          }
          part = (double)pf;
          stg16(DQKV + pix_index(b, p, n, H, W, unf) * ldq + cg * 8, pack8(dk));
        }
        for (int o = 1; o < 32 && o < cgs; o <<= 1) {
          const double t = __shfl_down_sync(0xffffffffu, part, o);
          if (lane + o <= seg_hi) part += t;
        }
        if (real && lane == seg_lo) s_dsp[piece * N + n] = part;
      }
    }
    if (grp < ngrp) {
#pragma unroll
      for (int j = 0; j < 8; ++j) s_part[grp * d + cg * 8 + j] = dbk[j];
    }
  }
  __syncthreads();
  for (int n = tid; n < N; n += blockDim.x) {
    double t = 0.0;
    for (int q = 0; q < npc; ++q) t += s_dsp[q * N + n];
    s_dsp[n] = t;  // slot q = 0 of row n: read only by this thread
  }
  if (dbias) {
    for (int i = tid; i < d; i += blockDim.x) {
      double t = 0.0;
      for (int gq = 0; gq < ngrp; ++gq) t += (double)s_part[gq * d + i];
      s_dbk[i] = t;
    }
  }
  __syncthreads();
  const double* s_ds = s_dsp;
  // dq = s * (ds - sum_n ds*s); written with the zero pad of the last 16-byte chunk
  float ldot = 0.f;
  for (int n = tid; n < N; n += blockDim.x) ldot += (float)s_ds[n] * s_s[n];
  const float dot = block_reduce_sum(ldot, ws);
  float ldq_sum = 0.f;
  for (int n = tid; n < N; n += blockDim.x) {
    const int64_t m = pix_index(b, p, n, H, W, unf);
    float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    f[0] = bf16_round(s_s[n] * ((float)s_ds[n] - dot));
    ldq_sum += f[0];
    for (int c = 2 * d; c < ldq; c += 8) {
      stg16(DQKV + m * ldq + c, pack8(f));
      f[0] = 0.f;
    }
  }
  if (dbias) {
    const float dq_sum = block_reduce_sum(ldq_sum, ws);
    for (int i = tid; i < d; i += blockDim.x) { atomicAdd(dbias + i, s_dbk[i]); atomicAdd(dbias + d + i, s_dbv[i]); }
    if (tid == 0) atomicAdd(dbias + 2 * d, (double)dq_sum);
  }
}

}  // namespace

static int check_common(const char* who, int ldq, int B, int H, int W, int d, int patch) {
  CVB_CHECK(B > 0 && H > 0 && W > 0 && d > 0, "%s: bad shape", who);
  CVB_CHECK((patch == 2 && H % 2 == 0 && W % 2 == 0) || patch == 0,
            "%s: patch must be 2 (folded feature map, even H, W) or 0 (unfolded [B, P=H, N=W] matrix); got patch=%d H=%d W=%d", who, patch, H, W);
  CVB_CHECK(d % 8 == 0 && d <= 8 * NT && ldq % 8 == 0 && ldq >= 2 * d + 8, "%s: need d %% 8 == 0 and ldq >= 2d+8 (d=%d ldq=%d)", who, d, ldq);
  return 0;
}

static int linattn_fwd_impl(const void* QKV, int ldq, int B, int H, int W, int d, int patch, const void* VX, int ldvx, int Nv, void* O, int ldo,
                            float* S, float* CTX, cvb_stream_t stream) {
  if (check_common("cvb_linattn_fwd", ldq, B, H, W, d, patch)) return 1;
  CVB_CHECK(QKV && O && S && CTX && ldo % 8 == 0 && ldo >= d, "cvb_linattn_fwd: bad arguments");
  const int N = patch == 0 ? W : (H / 2) * (W / 2);
  const int P = patch == 0 ? H : 4;
  if (VX == nullptr) { VX = QKV; ldvx = ldq; Nv = N; }
  CVB_CHECK(VX == QKV || patch == 0, "cvb_linattn_fwd: cross-attention needs the unfolded layout (patch = 0)");
  CVB_CHECK(ldvx % 8 == 0 && ldvx >= 2 * d && Nv > 0, "cvb_linattn_fwd: bad value tensor");
  const int nthreads = NT;  // a multiple of 32; threads beyond (d/8)*(NT/(d/8)) idle in the channel-grouped loops
  size_t smem = (size_t)(N + d + (size_t)(NT / (d / 8)) * d) * sizeof(float);
  CVB_CHECK(smem <= 200 * 1024, "cvb_linattn_fwd: N=%d too large", N);
  static bool attr = false;
  if (!attr) { CVB_CUDA(cudaFuncSetAttribute(linattn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  CVB_CUDA(cvb_launch(linattn_fwd_kernel, B * P, nthreads, smem, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(QKV), ldq, H, W, d,
                      static_cast<bf16*>(O), ldo, S, CTX, patch == 0 ? 1 : 0, static_cast<const bf16*>(VX), ldvx, Nv));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_linattn_fwd(const void* QKV, int ldq, int B, int H, int W, int d, int patch, void* O, int ldo, float* S, float* CTX,
                               cvb_stream_t stream) {
  return linattn_fwd_impl(QKV, ldq, B, H, W, d, patch, nullptr, 0, 0, O, ldo, S, CTX, stream);
}

extern "C" int cvb_linattn_cross_fwd(const void* QK_prev, int ldq, int B, int P, int M, int d, const void* V_x, int ldv, int N, void* O, int ldo,
                                     float* S, float* CTX, cvb_stream_t stream) {
  CVB_CHECK(V_x != nullptr, "cvb_linattn_cross_fwd: bad arguments");
  return linattn_fwd_impl(QK_prev, ldq, B, P, M, d, 0, V_x, ldv, N, O, ldo, S, CTX, stream);
}

static int linattn_bwd_impl(const void* QKV, int ldq, const void* DO, int ldo, const float* S, const float* CTX, int B, int H, int W, int d, int patch,
                            const void* VX, int ldvx, int Nv, void* DQKV, void* DVX, float* dbias, cvb_stream_t stream) {
  if (check_common("cvb_linattn_bwd", ldq, B, H, W, d, patch)) return 1;
  CVB_CHECK(QKV && DO && S && CTX && DQKV && ldo % 8 == 0 && ldo >= d, "cvb_linattn_bwd: bad arguments");
  const int N = patch == 0 ? W : (H / 2) * (W / 2);
  const int P = patch == 0 ? H : 4;
  if (VX == nullptr) { VX = QKV; ldvx = ldq; Nv = N; DVX = DQKV; }
  CVB_CHECK(VX == QKV || patch == 0, "cvb_linattn_bwd: cross-attention needs the unfolded layout (patch = 0)");
  CVB_CHECK(DVX && ldvx % 8 == 0 && ldvx >= 2 * d && Nv > 0, "cvb_linattn_bwd: bad value tensor");
  const int nthreads = NT;
  const int cgs = d / 8;
  size_t smem = (size_t)(la_pieces(cgs) * N + 3 * d) * sizeof(double) + (size_t)(2 * (NT / cgs) * d + N + d) * sizeof(float);
  CVB_CHECK(smem <= 200 * 1024, "cvb_linattn_bwd: N=%d too large", N);
  static bool attr = false;
  if (!attr) { CVB_CUDA(cudaFuncSetAttribute(linattn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* ws = nullptr;  // the CTAs' bias-gradient partials meet in fp64 (order-independent), added to dbias afterwards
  if (dbias && cvb_det_alloc(&ws, (size_t)2 * d + 1, st)) return 2;
  CVB_CUDA(cvb_launch(linattn_bwd_kernel, B * P, nthreads, smem, st, static_cast<const bf16*>(QKV), ldq,
                      static_cast<const bf16*>(DO), ldo, S, CTX, H, W, d, static_cast<bf16*>(DQKV), ws, patch == 0 ? 1 : 0,
                      static_cast<const bf16*>(VX), ldvx, Nv, static_cast<bf16*>(DVX)));
  CVB_LAUNCH_CHECK();
  if (!dbias) return 0;
  if (cvb_det_add(ws, dbias, 1, 2 * d + 1, 2 * d + 1, st)) return 2;
  return cvb_det_free(ws, st);
}

extern "C" int cvb_linattn_bwd(const void* QKV, int ldq, const void* DO, int ldo, const float* S, const float* CTX, int B, int H, int W, int d, int patch,
                               void* DQKV, float* dbias, cvb_stream_t stream) {
  return linattn_bwd_impl(QKV, ldq, DO, ldo, S, CTX, B, H, W, d, patch, nullptr, 0, 0, DQKV, nullptr, dbias, stream);
}

extern "C" int cvb_linattn_cross_bwd(const void* QK_prev, int ldq, const void* V_x, int ldv, const void* DO, int ldo, const float* S, const float* CTX,
                                     int B, int P, int M, int N, int d, void* DQK_prev, void* DV_x, float* dbias, cvb_stream_t stream) {
  CVB_CHECK(V_x != nullptr && DV_x != nullptr, "cvb_linattn_cross_bwd: bad arguments");
  return linattn_bwd_impl(QK_prev, ldq, DO, ldo, S, CTX, B, P, M, d, 0, V_x, ldv, N, DQK_prev, DV_x, dbias, stream);
}
