// Dropout / stochastic depth on the residual stream (cvnets/layers/dropout.py == nn.Dropout; torchvision.ops.StochasticDepth(mode="row") as used by
// cvnets/modules/transformer.py:97-100,139-156), sm_90a.
//
//   forward   Y[m, c] = R[m, c] + V[m, c] * e(m, c) * r(m / rows_per_sample)        (R optional)
//   backward  DV[m, c] = DY[m, c] * e(m, c) * r(...)                                   (the gradient of R is DY itself)
//   e = Bernoulli(1 - p) / (1 - p) per element,   r = Bernoulli(1 - p_row) / (1 - p_row) per sample
//
// The masks are never stored: they are a counter-based hash (splitmix64 finaliser) of a 64-bit KEY and the element / sample index, so the
// backward regenerates exactly the forward's mask from the key.  The key lives in device memory and is drawn by cvb_rng_next from a
// (seed, counter) state that the kernel itself advances -- a CUDA graph that contains the step therefore draws fresh masks on every replay
// (the same mechanism as torch's philox offset under graph capture, without a host round trip).
#include "common.cuh"

namespace {

constexpr int DR_NT = 256;

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__global__ void rng_next_kernel(unsigned long long* __restrict__ state, unsigned long long* __restrict__ key_out) {
  pdl_wait();
  pdl_trigger();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const uint64_t seed = state[0], ctr = state[1];
    key_out[0] = mix64(seed ^ mix64(ctr));
    state[1] = ctr + 1;
  }
}

struct DropArgs {
  int64_t ngroups;   // groups of 8 elements
  int C;             // row length (elements)
  int rows_per_sample;
  uint32_t thresh;   // keep iff u16 < thresh  (thresh = round((1 - p) * 65536); 65536 keeps everything)
  float scale;       // 1 / (1 - p)
  uint32_t row_thresh;  // keep the sample iff u24 < row_thresh
  float row_scale;
};

// factor of the 8 elements of group g (row m = g * 8 / C)
__device__ __forceinline__ void drop_factors(uint64_t key, int64_t g, const DropArgs& a, float* f) {
  float rowf = 1.0f;
  if (a.row_thresh < (1u << 24)) {
    const int64_t sample = (g * 8 / a.C) / a.rows_per_sample;
    const uint32_t u = (uint32_t)(mix64(key ^ 0xD1B54A32D192ED03ull ^ ((uint64_t)sample << 1)) >> 40);
    rowf = (u < a.row_thresh) ? a.row_scale : 0.f;
  }
  if (a.thresh >= 65536u) {
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = rowf;
    return;
  }
  const uint64_t r0 = mix64(key + 2 * (uint64_t)g), r1 = mix64(key + 2 * (uint64_t)g + 1);
  const float s = a.scale * rowf;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    f[e] = (((uint32_t)(r0 >> (16 * e)) & 0xFFFFu) < a.thresh) ? s : 0.f;
    f[4 + e] = (((uint32_t)(r1 >> (16 * e)) & 0xFFFFu) < a.thresh) ? s : 0.f;
  }
}

// Y = R + V * factor   (R may be null);   the backward is the same kernel with V = DY, R = null
__global__ void __launch_bounds__(DR_NT) dropout_kernel(const bf16* __restrict__ V, const bf16* __restrict__ R, bf16* __restrict__ Y,
                                                        const unsigned long long* __restrict__ key_ptr, const DropArgs a) {
  pdl_wait();
  pdl_trigger();
  const uint64_t key = key_ptr[0];
  for (int64_t g = (int64_t)blockIdx.x * DR_NT + threadIdx.x; g < a.ngroups; g += (int64_t)gridDim.x * DR_NT) {
    float v[8], f[8];
    unpack8(ldg16_stream(V + g * 8), v);
    drop_factors(key, g, a, f);
    if (R) {
      float r[8];
      unpack8(ldg16_stream(R + g * 8), r);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = fmaf(v[e], f[e], r[e]);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] *= f[e];
    }
    stg16(Y + g * 8, pack8(v));
  }
}

int make_args(const char* who, int64_t M, int C, int rows_per_sample, float p, float p_row, DropArgs* a) {
  CVB_CHECK(M > 0 && C > 0 && C % 8 == 0, "%s: bad shape M=%lld C=%d (C %% 8 == 0)", who, (long long)M, C);
  CVB_CHECK(p >= 0.f && p < 1.f && p_row >= 0.f && p_row < 1.f, "%s: probabilities must be in [0, 1): p=%g p_row=%g", who, p, p_row);
  CVB_CHECK(p_row == 0.f || rows_per_sample > 0, "%s: stochastic depth needs rows_per_sample", who);
  a->ngroups = M * C / 8;
  a->C = C;
  a->rows_per_sample = rows_per_sample > 0 ? rows_per_sample : 1;
  double keep = 1.0 - (double)p;
  uint32_t th = (uint32_t)(keep * 65536.0 + 0.5);
  if (p > 0.f && th >= 65536u) th = 65535u;
  a->thresh = p > 0.f ? th : 65536u;
  a->scale = (float)(1.0 / keep);
  double keep_r = 1.0 - (double)p_row;
  uint32_t rt = (uint32_t)(keep_r * 16777216.0 + 0.5);
  if (p_row > 0.f && rt >= (1u << 24)) rt = (1u << 24) - 1;
  a->row_thresh = p_row > 0.f ? rt : (1u << 24);
  a->row_scale = (float)(1.0 / keep_r);
  return 0;
}

int launch(const void* V, const void* R, void* Y, const void* key, const DropArgs& a, cudaStream_t st) {
  int64_t blocks = (a.ngroups + DR_NT - 1) / DR_NT;
  const int64_t cap = (int64_t)cvb_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  CVB_CUDA(cvb_launch(dropout_kernel, (int)blocks, DR_NT, 0, st, static_cast<const bf16*>(V), static_cast<const bf16*>(R), static_cast<bf16*>(Y),
                      static_cast<const unsigned long long*>(key), a));
  return 0;
}

}  // namespace

extern "C" int cvb_rng_next(void* state, void* key_out, cvb_stream_t stream) {
  CVB_CHECK(state && key_out, "cvb_rng_next: null pointer");
  CVB_CUDA(cvb_launch(rng_next_kernel, 1, 32, 0, static_cast<cudaStream_t>(stream), static_cast<unsigned long long*>(state),
                      static_cast<unsigned long long*>(key_out)));
  return 0;
}

extern "C" int cvb_dropout_fwd(const void* V, const void* R, void* Y, int64_t M, int C, int rows_per_sample, float p, float p_row, const void* key,
                               cvb_stream_t stream) {
  DropArgs a;
  if (make_args("cvb_dropout_fwd", M, C, rows_per_sample, p, p_row, &a)) return 1;
  CVB_CHECK(V && Y && key && cvb_aligned16(V) && cvb_aligned16(Y) && (!R || cvb_aligned16(R)), "cvb_dropout_fwd: null / misaligned operand");
  return launch(V, R, Y, key, a, static_cast<cudaStream_t>(stream));
}

extern "C" int cvb_dropout_bwd(const void* DY, void* DV, int64_t M, int C, int rows_per_sample, float p, float p_row, const void* key,
                               cvb_stream_t stream) {
  DropArgs a;
  if (make_args("cvb_dropout_bwd", M, C, rows_per_sample, p, p_row, &a)) return 1;
  CVB_CHECK(DY && DV && key && cvb_aligned16(DY) && cvb_aligned16(DV), "cvb_dropout_bwd: null / misaligned operand");
  return launch(DY, nullptr, DV, key, a, static_cast<cudaStream_t>(stream));
}
