// Device helpers shared by the two head_dim-64 wgmma attention families (mha_tc.cu: register-resident, S <= 256; mha_long.cu: streaming).
// Both read every operand as [64 rows x 64 ch] bf16 SWIZZLE_128B images and keep scores and LSE in the exp2 domain, so these define
// the operand images and the LSE convention for both: a change here changes both families together.
#pragma once
#include "common.cuh"

#include <math_constants.h>

constexpr float LOG2E = 1.4426950408889634f;
constexpr int BOX64 = 64 * 128;  // bytes of a [64 rows x 64 ch] image

__device__ __forceinline__ uint64_t desc_k(uint32_t saddr) { return wgmma_desc(saddr, 16, 1024, WG_SW128); }      // K-major: +32 B per k-step
__device__ __forceinline__ uint64_t desc_mn(uint32_t saddr) { return wgmma_desc(saddr, BOX64, 1024, WG_SW128); }  // MN-major: +2 KB per k-step
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// additive mask term (exp2 domain) of score (q, t), t < S; -inf for padded keys
__device__ __forceinline__ float mask_add(const float* amask, const uint8_t* kpm, int b, int S, int q, int t) {
  if (kpm && kpm[(size_t)b * S + t]) return -CUDART_INF_F;
  if (amask && q < S) return amask[((size_t)b * S + q) * S + t] * LOG2E;
  return 0.f;
}
// accumulator columns [16 kk, 16 kk + 16) of an m64n64 fp32 result, scaled, as the bf16 A operand of k-step kk
__device__ __forceinline__ void to_a_frag(const float* acc, int kk, uint32_t* a) {
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = pack_bf162(acc[8 * kk + 2 * i], acc[8 * kk + 2 * i + 1]);
}
// m64n64 fp32 accumulator * mul -> bf16 rows row0 + r (r < 64, row0 + r < S) of a [.. x 64] global matrix with leading dimension ld
__device__ __forceinline__ void store_acc(bf16* dst, int ld, const float* acc, float mul, int row0, int S) {
  const int lane = threadIdx.x & 31, r = ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + r + 8 * h;
    if (row < S) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(dst + (size_t)row * ld + 8 * j + 2 * (lane & 3)) = pack_bf162(acc[4 * j + 2 * h] * mul, acc[4 * j + 2 * h + 1] * mul);
    }
  }
}
