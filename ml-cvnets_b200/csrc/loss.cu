// Classification loss of the training step (loss_fn/classification/cross_entropy.py:74-95 of the reference ==
// F.cross_entropy(prediction, target, ignore_index, label_smoothing)) as two launches, plus two small step utilities:
//   cvb_ce_fwd : per-row log-sum-exp (saved) + the mean label-smoothed loss (one CTA; deterministic reduction order)
//   cvb_ce_bwd : dlogits = gscale * (softmax - target distribution) / n_valid, written as the padded bf16 matrix the classifier's
//                input-/weight-gradient GEMMs read (pad columns zeroed); gscale = grad_out * loss_scale, both device scalars
//   cvb_cast_f64_f32 : batched fp64 -> fp32 scatter (statistics accumulators -> gradient slices), one launch per module
#include "common.cuh"

namespace {

constexpr int LNT = 1024;

// one warp per row: max, sum of exp, sum of logits (for the smoothing term), the target logit
__global__ void __launch_bounds__(LNT) ce_fwd_kernel(const bf16* __restrict__ logits, int ld, int B, int C, const int64_t* __restrict__ target,
                                                     int ignore_index, float smoothing, float* __restrict__ lse, float* __restrict__ loss_out,
                                                     float* __restrict__ nvalid_out, const float* __restrict__ mix, const float* __restrict__ scale_param) {
  pdl_wait();
  pdl_trigger();
  __shared__ float s_loss[LNT / 32], s_cnt[LNT / 32];
  // CLIP (contrastive_loss_clip.py:74-79, clip.py _exponentiate_and_clip_logits): logits = clamp(exp(logit_scale), 0, 100) * raw similarities
  const float sc = scale_param ? fminf(__expf(scale_param[0]), 100.0f) : 1.0f;
  // batch mixing (RandomMixup / RandomCutmix targets, image_torch.py:119-137): target distribution = lam*onehot(y[r]) + (1-lam)*onehot(y[r-1])
  const bool mixing = mix != nullptr && mix[0] != 0.f;
  const float lam = mixing ? mix[1] : 1.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float loss = 0.f, cnt = 0.f;
  for (int r = warp; r < B; r += LNT / 32) {
    const bf16* row = logits + (size_t)r * ld;
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, sc * __bfloat162float(row[c]));
    mx = warp_max(mx);
    float se = 0.f, sl = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float v = sc * __bfloat162float(row[c]);
      se += __expf(v - mx);
      sl += v;
    }
    se = warp_sum(se);
    sl = warp_sum(sl);
    const float l = mx + __logf(se);
    if (lane == 0) {
      lse[r] = l;
      const int64_t t = target[r];
      if (t != (int64_t)ignore_index && t >= 0 && t < C) {
        // label smoothing (torch): (1-eps) * nll(target) + eps/C * sum_c nll(c)
        float nll_t = l - sc * __bfloat162float(row[t]);
        if (mixing) {
          const int64_t t2 = target[r == 0 ? B - 1 : r - 1];
          if (t2 >= 0 && t2 < C) nll_t = lam * nll_t + (1.0f - lam) * (l - sc * __bfloat162float(row[t2]));
        }
        const float nll_all = (float)C * l - sl;
        loss += (1.0f - smoothing) * nll_t + smoothing / (float)C * nll_all;
        cnt += 1.0f;
      }
    }
  }
  if (lane == 0) { s_loss[warp] = loss; s_cnt[warp] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < LNT / 32; ++w) { a += s_loss[w]; b += s_cnt[w]; }
    loss_out[0] = b > 0.f ? a / b : 0.f;
    nvalid_out[0] = b;
  }
}

__global__ void __launch_bounds__(256) ce_bwd_kernel(const bf16* __restrict__ logits, int ld, int B, int C, const int64_t* __restrict__ target,
                                                     int ignore_index, float smoothing, const float* __restrict__ lse,
                                                     const float* __restrict__ nvalid, const float* __restrict__ gout, const float* __restrict__ gscale,
                                                     bf16* __restrict__ dlogits, int ldd, const float* __restrict__ mix, const float* __restrict__ scale_param,
                                                     float* __restrict__ dscale_param) {
  pdl_wait();
  pdl_trigger();
  __shared__ float s_ds[8];
  const float se_raw = scale_param ? __expf(scale_param[0]) : 1.0f;
  const float sc = scale_param ? fminf(se_raw, 100.0f) : 1.0f;
  float ds = 0.f;  // sum_c dL/dv * raw logit   (v = sc * raw)
  const int r = blockIdx.x;
  const int64_t t = target[r];
  const bool mixing = mix != nullptr && mix[0] != 0.f;
  const float lam = mixing ? mix[1] : 1.f;
  const int64_t t2 = mixing ? target[r == 0 ? B - 1 : r - 1] : (int64_t)-1;
  const bool valid = (t != (int64_t)ignore_index && t >= 0 && t < C);
  float g = (gout ? gout[0] : 1.0f) * (gscale ? gscale[0] : 1.0f);
  const float nv = nvalid[0];
  g = (valid && nv > 0.f) ? g / nv : 0.f;
  const float l = lse[r];
  const bf16* row = logits + (size_t)r * ld;
  bf16* drow = dlogits + (size_t)r * ldd;
  const float off = smoothing / (float)C;
  for (int c = threadIdx.x; c < ldd; c += blockDim.x) {
    float d = 0.f;
    if (c < C) {
      const float x = __bfloat162float(row[c]);
      const float p = __expf(sc * x - l);
      d = g * (p - off - (1.0f - smoothing) * (((int64_t)c == t ? lam : 0.f) + ((int64_t)c == t2 ? 1.0f - lam : 0.f)));
      ds = fmaf(d, x, ds);
      d *= sc;  // gradient w.r.t. the RAW similarity
    }
    drow[c] = __float2bfloat16_rn(d);
  }
  if (dscale_param != nullptr) {  // d logit_scale = exp(logit_scale) * sum dv * raw   (0 where the clamp is active)
    ds = warp_sum(ds);
    if ((threadIdx.x & 31) == 0) s_ds[threadIdx.x >> 5] = ds;
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += s_ds[w];
      if (se_raw < 100.0f) atomicAdd(dscale_param, tot * se_raw);
    }
  }
}

struct CastDesc {
  const double* src;
  float* dst;
  int n;
  int pad;
};

__global__ void __launch_bounds__(256) cast_f64_f32_kernel(const CastDesc* __restrict__ descs) {
  pdl_wait();
  pdl_trigger();
  const CastDesc d = descs[blockIdx.y];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < d.n; i += gridDim.x * blockDim.x) d.dst[i] = (float)d.src[i];
}

}  // namespace

extern "C" int cvb_ce_fwd(const void* logits, int ld, int B, int C, const int64_t* target, int ignore_index, float label_smoothing, float* lse,
                          float* loss, float* n_valid, const float* mix, const float* logit_scale, cvb_stream_t stream) {
  CVB_CHECK(logits && target && lse && loss && n_valid && B > 0 && C > 0 && ld >= C, "cvb_ce_fwd: bad arguments");
  CVB_CUDA(cvb_launch(ce_fwd_kernel, 1, LNT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(logits), ld, B, C, target, ignore_index,
                      label_smoothing, lse, loss, n_valid, mix, logit_scale));
  return 0;
}

extern "C" int cvb_ce_bwd(const void* logits, int ld, int B, int C, const int64_t* target, int ignore_index, float label_smoothing, const float* lse,
                          const float* n_valid, const float* grad_out, const float* grad_scale, void* dlogits, int ldd, const float* mix,
                          const float* logit_scale, float* dlogit_scale, cvb_stream_t stream) {
  CVB_CHECK(logits && target && lse && n_valid && dlogits && B > 0 && C > 0 && ld >= C && ldd >= C, "cvb_ce_bwd: bad arguments");
  CVB_CUDA(cvb_launch(ce_bwd_kernel, B, 256, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(logits), ld, B, C, target, ignore_index,
                      label_smoothing, lse, n_valid, grad_out, grad_scale, static_cast<bf16*>(dlogits), ldd, mix, logit_scale, dlogit_scale));
  return 0;
}

extern "C" int cvb_cast_f64_f32(const cvb_cast_desc* descs_device, int n_desc, int max_n, cvb_stream_t stream) {
  CVB_CHECK(descs_device && n_desc > 0 && max_n > 0, "cvb_cast_f64_f32: bad arguments");
  static_assert(sizeof(CastDesc) == sizeof(cvb_cast_desc), "descriptor layout");
  int gx = (max_n + 255) / 256;
  if (gx > 16) gx = 16;
  CVB_CUDA(cvb_launch(cast_f64_f32_kernel, dim3(gx, n_desc), 256, 0, static_cast<cudaStream_t>(stream), reinterpret_cast<const CastDesc*>(descs_device)));
  return 0;
}

namespace {
__global__ void __launch_bounds__(256) transpose_bf16_kernel(const bf16* __restrict__ X, bf16* __restrict__ Y, int R, int C) {
  pdl_wait();
  pdl_trigger();
  __shared__ bf16 tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8)
    if (by + j < R && bx + tx < C) tile[j][tx] = X[(size_t)(by + j) * C + bx + tx];
  __syncthreads();
  for (int j = ty; j < 32; j += 8)
    if (bx + j < C && by + tx < R) Y[(size_t)(bx + j) * R + by + tx] = tile[tx][j];
}
__global__ void __launch_bounds__(256) add_bf16_f32_kernel(const bf16* __restrict__ A, const float* __restrict__ Bf, bf16* __restrict__ OUT, int64_t n) {
  pdl_wait();
  pdl_trigger();
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256)
    OUT[i] = __float2bfloat16_rn((A ? __bfloat162float(A[i]) : 0.f) + Bf[i]);
}
}  // namespace

extern "C" int cvb_transpose_bf16(const void* X, void* Y, int R, int C, cvb_stream_t stream) {
  CVB_CHECK(X && Y && R > 0 && C > 0, "cvb_transpose_bf16: bad arguments");
  CVB_CUDA(cvb_launch(transpose_bf16_kernel, dim3((C + 31) / 32, (R + 31) / 32), 256, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(X),
                      static_cast<bf16*>(Y), R, C));
  return 0;
}

extern "C" int cvb_add_bf16_f32(const void* A, const float* B, void* OUT, int64_t n, cvb_stream_t stream) {
  CVB_CHECK(B && OUT && n > 0, "cvb_add_bf16_f32: bad arguments");
  int64_t g = (n + 255) / 256;
  if (g > 4096) g = 4096;
  CVB_CUDA(cvb_launch(add_bf16_f32_kernel, (int)g, 256, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(A), B, static_cast<bf16*>(OUT), n));
  return 0;
}

extern "C" int cvb_memset_zero(void* ptr, int64_t bytes, cvb_stream_t stream) {
  CVB_CHECK(ptr && bytes > 0, "cvb_memset_zero: bad arguments");
  CVB_CUDA(cudaMemsetAsync(ptr, 0, (size_t)bytes, static_cast<cudaStream_t>(stream)));
  return 0;
}
