// Squeeze-excitation channel scaling (cvnets/modules/squeeze_excitation.py:82-83: `x * self.se_layer(x)`), sm_90a.
//
//   forward   Y[b, p, c] = X[b, p, c] * S[b, c]                       X, Y: bf16 channels-last [B, HW, C]; S: bf16 [B, C]
//   backward  DX[b, p, c] = DY[b, p, c] * S[b, c];   DS[b, c] += sum_p DY[b, p, c] * X[b, p, c]      (DS fp32, zero-initialised by the caller)
//
// Pure bandwidth: one pass over the map with 16-byte accesses.  A CTA owns a strip of pixels of one sample; a thread keeps one 8-channel
// group, so its scale vector and its DS partial stay in registers; partials meet in shared memory and leave with one atomic per
// (CTA, channel).  The pooled vector / the two 1x1 convs of the SE unit are the library's pool and GEMM kernels.
#include "common.cuh"

namespace {

constexpr int SE_NT = 256;

// grid: (strips, B).  Thread t: channel group t % cgs, pixel lane t / cgs (cgs = C / 8 <= SE_NT)
__global__ void __launch_bounds__(SE_NT) se_scale_fwd_kernel(const bf16* __restrict__ X, const bf16* __restrict__ S, bf16* __restrict__ Y, int HW, int C,
                                                             int rows_per_cta) {
  pdl_wait();
  pdl_trigger();
  const int cgs = C / 8, lanes = SE_NT / cgs;
  const int cg = threadIdx.x % cgs, pl = threadIdx.x / cgs;
  if (pl >= lanes) return;
  const int b = blockIdx.y;
  float s[8];
  unpack8(ldg16(S + (size_t)b * C + cg * 8), s);
  const int p0 = blockIdx.x * rows_per_cta, p1 = min(HW, p0 + rows_per_cta);
  for (int p = p0 + pl; p < p1; p += lanes) {
    const size_t off = ((size_t)b * HW + p) * C + cg * 8;
    float f[8];
    unpack8(ldg16_stream(X + off), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] *= s[e];
    stg16(Y + off, pack8(f));
  }
}

__global__ void __launch_bounds__(SE_NT) se_scale_bwd_kernel(const bf16* __restrict__ DY, const bf16* __restrict__ X, const bf16* __restrict__ S,
                                                             bf16* __restrict__ DX, float* __restrict__ DS, int HW, int C, int rows_per_cta) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float s_ds[];  // [C]
  for (int c = threadIdx.x; c < C; c += SE_NT) s_ds[c] = 0.f;
  __syncthreads();
  const int cgs = C / 8, lanes = SE_NT / cgs;
  const int cg = threadIdx.x % cgs, pl = threadIdx.x / cgs;
  const int b = blockIdx.y;
  if (pl < lanes) {
    float s[8], acc[8];
    unpack8(ldg16(S + (size_t)b * C + cg * 8), s);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = 0.f;
    const int p0 = blockIdx.x * rows_per_cta, p1 = min(HW, p0 + rows_per_cta);
    for (int p = p0 + pl; p < p1; p += lanes) {
      const size_t off = ((size_t)b * HW + p) * C + cg * 8;
      float g[8], x[8];
      unpack8(ldg16_stream(DY + off), g);
      unpack8(ldg16_stream(X + off), x);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        acc[e] = fmaf(g[e], x[e], acc[e]);
        g[e] *= s[e];
      }
      stg16(DX + off, pack8(g));
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) atomicAdd(&s_ds[cg * 8 + e], acc[e]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += SE_NT) atomicAdd(DS + (size_t)b * C + c, s_ds[c]);
}

int se_geometry(const char* who, int B, int HW, int C, int* rows_per_cta, int* strips) {
  CVB_CHECK(B > 0 && HW > 0 && C > 0 && C % 8 == 0 && C / 8 <= SE_NT, "%s: bad shape B=%d HW=%d C=%d (C %% 8 == 0, C <= %d)", who, B, HW, C, 8 * SE_NT);
  // ~4 waves of CTAs over the SMs, at least 32 pixels per CTA
  int s = (4 * cvb_num_sms() + B - 1) / B;
  int rpc = (HW + s - 1) / s;
  if (rpc < 32) rpc = 32;
  *rows_per_cta = rpc;
  *strips = (HW + rpc - 1) / rpc;
  return 0;
}

}  // namespace

extern "C" int cvb_se_scale_fwd(const void* X, const void* S, void* Y, int B, int HW, int C, cvb_stream_t stream) {
  int rpc, strips;
  if (se_geometry("cvb_se_scale_fwd", B, HW, C, &rpc, &strips)) return 1;
  CVB_CHECK(X && S && Y && cvb_aligned16(X) && cvb_aligned16(S) && cvb_aligned16(Y), "cvb_se_scale_fwd: null / misaligned operand");
  CVB_CUDA(cvb_launch(se_scale_fwd_kernel, dim3(strips, B), SE_NT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(X),
                      static_cast<const bf16*>(S), static_cast<bf16*>(Y), HW, C, rpc));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_se_scale_bwd(const void* DY, const void* X, const void* S, void* DX, float* DS, int B, int HW, int C, cvb_stream_t stream) {
  int rpc, strips;
  if (se_geometry("cvb_se_scale_bwd", B, HW, C, &rpc, &strips)) return 1;
  CVB_CHECK(DY && X && S && DX && DS && cvb_aligned16(DY) && cvb_aligned16(X) && cvb_aligned16(S) && cvb_aligned16(DX),
            "cvb_se_scale_bwd: null / misaligned operand");
  CVB_CUDA(cvb_launch(se_scale_bwd_kernel, dim3(strips, B), SE_NT, (size_t)C * sizeof(float), static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(DY), static_cast<const bf16*>(X), static_cast<const bf16*>(S), static_cast<bf16*>(DX), DS, HW, C, rpc));
  CVB_LAUNCH_CHECK();
  return 0;
}
