// CLIP zero-shot evaluation (cvnets/text_encoders/transformer.py:428-504, cvnets/models/multi_modal_img_text/clip.py:171-202,
// metrics/topk_accuracy.py), sm_90a.
//   cvb_zs_class_embed : per class, the caption features of the text tower's projection are L2-normalised in fp32, averaged over the
//                        captions in a fixed order and normalised again; written transposed as the fp32 [d, Cl] class table.  One warp
//                        owns a class (no atomics): the table is bitwise reproducible.
//   cvb_zs_logits_topk : fp32 logits = scale * img @ table, and top-1 / top-5 hit counts from the rank of the target's logit (the number
//                        of classes with a strictly greater logit), added into a device int64[2].  Integer adds: deterministic.
#include "common.cuh"

namespace {

constexpr int CE_WARPS = 4;      // classes per CTA of the class-embedding kernel
constexpr int CE_MAX_CHUNK = 4;  // 8-wide chunks per lane: d <= 4 * 256
constexpr int LT_THREADS = 256;
constexpr int LT_ROWS = 4;       // image rows per CTA of the logits kernel

__global__ void __launch_bounds__(CE_WARPS * 32) zs_class_embed_kernel(const bf16* __restrict__ X, int ldx, int R, const int* __restrict__ perm,
                                                                        int Cl, int M, int d, float* __restrict__ table) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * CE_WARPS + (threadIdx.x >> 5);
  if (c >= Cl) return;
  float acc[CE_MAX_CHUNK][8];
#pragma unroll
  for (int j = 0; j < CE_MAX_CHUNK; ++j)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[j][e] = 0.f;
  for (int m = 0; m < M; ++m) {
    const int r = perm[(int64_t)c * M + m];
    if (r < 0 || r >= R) continue;
    const bf16* x = X + (int64_t)r * ldx;
    float f[CE_MAX_CHUNK][8];
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < CE_MAX_CHUNK; ++j) {
      const int k = j * 256 + lane * 8;
      if (k < d) {
        unpack8(ldg16(x + k), f[j]);
#pragma unroll
        for (int e = 0; e < 8; ++e) q = __fmaf_rn(f[j][e], f[j][e], q);
      }
    }
    q = warp_sum(q);  // fixed butterfly: the same order for every caption and every run
    const float den = fmaxf(__fsqrt_rn(q), 1e-12f);  // F.normalize: x / max(||x||, eps)
#pragma unroll
    for (int j = 0; j < CE_MAX_CHUNK; ++j)
      if (j * 256 + lane * 8 < d)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[j][e] = __fadd_rn(acc[j][e], __fdiv_rn(f[j][e], den));
  }
  const float fm = (float)M;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < CE_MAX_CHUNK; ++j)
    if (j * 256 + lane * 8 < d)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        acc[j][e] = __fdiv_rn(acc[j][e], fm);  // the mean over the captions
        q = __fmaf_rn(acc[j][e], acc[j][e], q);
      }
  q = warp_sum(q);
  const float den = fmaxf(__fsqrt_rn(q), 1e-12f);
#pragma unroll
  for (int j = 0; j < CE_MAX_CHUNK; ++j) {
    const int k = j * 256 + lane * 8;
    if (k < d)
#pragma unroll
      for (int e = 0; e < 8; ++e) table[(int64_t)(k + e) * Cl + c] = __fdiv_rn(acc[j][e], den);
  }
}

// one fp32 dot product of an image row (shared memory) with a table column; the target's logit and every class's logit go through
// exactly this chain of fmas, so "strictly greater than the target" compares bitwise-consistent values
__device__ __forceinline__ float zs_dot(const float* __restrict__ img, const float* __restrict__ table, int d, int Cl, int c) {
  float a = 0.f;
  for (int k = 0; k < d; ++k) a = __fmaf_rn(img[k], table[(int64_t)k * Cl + c], a);
  return a;
}

__global__ void __launch_bounds__(LT_THREADS) zs_logits_topk_kernel(const bf16* __restrict__ img, int ldi, const float* __restrict__ table, int B,
                                                                     int d, int Cl, float scale, const int64_t* __restrict__ targets,
                                                                     float* __restrict__ logits, unsigned long long* __restrict__ hits) {
  extern __shared__ float s_img[];  // [LT_ROWS][d]
  __shared__ float s_tl[LT_ROWS];
  __shared__ int s_tgt[LT_ROWS];
  __shared__ unsigned int s_rank[LT_ROWS];
  pdl_wait();
  pdl_trigger();
  const int b0 = blockIdx.x * LT_ROWS;
  for (int i = threadIdx.x; i < LT_ROWS * d; i += LT_THREADS) {
    const int r = i / d, k = i - r * d;
    s_img[i] = (b0 + r < B) ? __bfloat162float(img[(int64_t)(b0 + r) * ldi + k]) : 0.f;
  }
  const bool rank = targets != nullptr && hits != nullptr;
  if (threadIdx.x < LT_ROWS) {
    const int b = b0 + threadIdx.x;
    int t = -1;
    if (rank && b < B) {
      const int64_t tv = targets[b];
      t = (tv >= 0 && tv < Cl) ? (int)tv : -1;  // a target outside [0, Cl) is a miss
    }
    s_tgt[threadIdx.x] = t;
    s_rank[threadIdx.x] = 0u;
  }
  __syncthreads();
  if (rank && threadIdx.x < LT_ROWS && s_tgt[threadIdx.x] >= 0)
    s_tl[threadIdx.x] = __fmul_rn(scale, zs_dot(s_img + threadIdx.x * d, table, d, Cl, s_tgt[threadIdx.x]));
  __syncthreads();
  unsigned int above[LT_ROWS];
#pragma unroll
  for (int i = 0; i < LT_ROWS; ++i) above[i] = 0u;
  for (int c = threadIdx.x; c < Cl; c += LT_THREADS) {
    float a[LT_ROWS];
#pragma unroll
    for (int i = 0; i < LT_ROWS; ++i) a[i] = 0.f;
    for (int k = 0; k < d; ++k) {
      const float t = table[(int64_t)k * Cl + c];
#pragma unroll
      for (int i = 0; i < LT_ROWS; ++i) a[i] = __fmaf_rn(s_img[i * d + k], t, a[i]);
    }
#pragma unroll
    for (int i = 0; i < LT_ROWS; ++i) {
      const float v = __fmul_rn(scale, a[i]);
      if (b0 + i < B) {
        if (logits) logits[(int64_t)(b0 + i) * Cl + c] = v;
        if (rank && s_tgt[i] >= 0 && v > s_tl[i]) ++above[i];
      }
    }
  }
  if (rank) {
#pragma unroll
    for (int i = 0; i < LT_ROWS; ++i) {
      const unsigned int w = __reduce_add_sync(0xffffffffu, above[i]);
      if ((threadIdx.x & 31) == 0 && w) atomicAdd(&s_rank[i], w);
    }
    __syncthreads();
    if (threadIdx.x < LT_ROWS && b0 + threadIdx.x < B && s_tgt[threadIdx.x] >= 0) {
      const unsigned int r = s_rank[threadIdx.x];
      if (r < 1u) atomicAdd(hits + 0, 1ull);
      if (r < 5u) atomicAdd(hits + 1, 1ull);
    }
  }
}

}  // namespace

extern "C" int cvb_zs_class_embed(const void* X, int ldx, int R, const int* perm, int Cl, int M, int d, float* table, cvb_stream_t stream) {
  CVB_CHECK(X && perm && table && R > 0 && Cl > 0 && M > 0 && d > 0 && d % 8 == 0 && d <= CE_MAX_CHUNK * 256 && ldx >= d && ldx % 8 == 0 &&
                cvb_aligned16(X),
            "cvb_zs_class_embed: bad arguments (d %% 8 == 0, d <= %d, ldx >= d, ldx %% 8 == 0, 16-byte aligned rows)", CE_MAX_CHUNK * 256);
  CVB_CUDA(cvb_launch(zs_class_embed_kernel, (Cl + CE_WARPS - 1) / CE_WARPS, CE_WARPS * 32, 0, static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(X), ldx, R, perm, Cl, M, d, table));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_zs_logits_topk(const void* img, int ldi, const float* table, int B, int d, int Cl, float scale, const int64_t* targets,
                                  float* logits, int64_t* hits, cvb_stream_t stream) {
  CVB_CHECK(img && table && B > 0 && d > 0 && d <= 4096 && ldi >= d && Cl > 0, "cvb_zs_logits_topk: bad arguments (d <= 4096, ldi >= d)");
  CVB_CHECK(logits || (targets && hits), "cvb_zs_logits_topk: nothing to compute (no logits output, no targets + hits)");
  const size_t smem = sizeof(float) * LT_ROWS * d;
  if (smem > 48 * 1024) CVB_CUDA(cudaFuncSetAttribute(zs_logits_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CVB_CUDA(cvb_launch(zs_logits_topk_kernel, (B + LT_ROWS - 1) / LT_ROWS, LT_THREADS, smem, static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(img), ldi, table, B, d, Cl, scale, targets, logits, reinterpret_cast<unsigned long long*>(hits)));
  CVB_LAUNCH_CHECK();
  return 0;
}
