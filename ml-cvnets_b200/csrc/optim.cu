// Per-step tail of Trainer.train_epoch (engine/training_engine.py:289-312) on FLAT fp32 buffers, two launches:
//   1. cvb_grad_norm : unscale (GradScaler, :290-292) + global L2 norm for clip_grad_norm_ (:293-295) + inf/nan detection
//   2. cvb_adamw_step: clip coefficient, decoupled-weight-decay AdamW (torch.optim.AdamW semantics: optim/adamw.py wrapper of the
//                      reference, cvnets/optim/adamw.py), GradScaler.step "skip on inf" and GradScaler.update (growth / backoff)
//      or cvb_sgd_step: the same around torch.optim.SGD with momentum / Nesterov / L2 weight decay (optim/sgd.py)
// State (all device resident, so the whole step stays one CUDA graph): partials[] = per-block (sum of squares, non-finite count) of the
// unscaled gradients, reduced in a fixed order (deterministic: data-parallel replicas stay bit-identical); stats[0..1] = those totals of the
// last step (for logging), stats[2] = 1 / loss_scale used by this step; scale[0] = loss scale,
// scale[1] = growth tracker; step[0] = optimizer step count (fp32); hp[0] = learning rate (device scalar: a scheduler writes it every
// iteration, scheduler.update_lr at engine/training_engine.py:246-249, without re-capturing the step's CUDA graph).
// Optional: the EMA of the weights (cvnets/misc/averaging_utils.py:43-55: ema = ema*(1-momentum) + momentum*param, every iteration)
// rides in the same pass, and grad_div folds DDP's division by the world size into the unscale.
#include "common.cuh"

namespace {

constexpr int ONT = 256;

__global__ void __launch_bounds__(ONT) grad_norm_kernel(const float* __restrict__ g, int64_t n, const float* __restrict__ scale, float grad_div,
                                                        float* stats, float* __restrict__ partials) {
  pdl_wait();
  pdl_trigger();
  __shared__ float s_sq[ONT / 32], s_bad[ONT / 32];
  const float inv = 1.0f / (scale[0] * grad_div);
  float sq = 0.f, bad = 0.f;
  const int64_t nvec = n >> 2;
  for (int64_t i = (int64_t)blockIdx.x * ONT + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * ONT) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(g) + i);
    const float a = v.x * inv, b = v.y * inv, c = v.z * inv, d = v.w * inv;
    sq = fmaf(a, a, fmaf(b, b, fmaf(c, c, fmaf(d, d, sq))));
    bad += (isfinite(a) ? 0.f : 1.f) + (isfinite(b) ? 0.f : 1.f) + (isfinite(c) ? 0.f : 1.f) + (isfinite(d) ? 0.f : 1.f);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int64_t i = nvec << 2; i < n; ++i) {
      const float a = g[i] * inv;
      sq = fmaf(a, a, sq);
      bad += isfinite(a) ? 0.f : 1.f;
    }
    stats[2] = inv;
  }
  sq = warp_sum(sq);
  bad = warp_sum(bad);
  if ((threadIdx.x & 31) == 0) { s_sq[threadIdx.x >> 5] = sq; s_bad[threadIdx.x >> 5] = bad; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < ONT / 32; ++w) { a += s_sq[w]; b += s_bad[w]; }
    // one slot per block, combined in a FIXED order by every block of the step kernel: the norm -- and with it the clip coefficient and
    // the update -- is bit-identical on every data-parallel rank (an atomic sum would let replicas drift apart by an ulp per step)
    partials[2 * blockIdx.x] = a;
    partials[2 * blockIdx.x + 1] = b;
  }
}

// ---- shared by the optimizer step kernels: fixed-order totals of grad_norm's partials, clip coefficient, the EMA of a skipped step and
// the last block's scalar bookkeeping (GradScaler.update, step count, statistics)
__device__ __forceinline__ void step_totals(const float* __restrict__ partials, int n_partials, float* s_tot) {
  if (threadIdx.x < 32) {  // fixed-order reduction of the per-block partial sums (same tree in every block and on every rank)
    float a = 0.f, b = 0.f;
    for (int i = threadIdx.x; i < n_partials; i += 32) { a += partials[2 * i]; b += partials[2 * i + 1]; }
    a = warp_sum(a);
    b = warp_sum(b);
    if (threadIdx.x == 0) { s_tot[0] = a; s_tot[1] = b; }
  }
  __syncthreads();
}

// unscale * clip: torch.nn.utils.clip_grad_norm_ (clip_coef clamped to 1); max_norm <= 0 = no clipping
__device__ __forceinline__ float grad_scale(float inv, float sumsq, float max_norm) {
  const float norm = sqrtf(sumsq);
  float coef = max_norm / (norm + 1e-6f);
  if (!(coef < 1.0f)) coef = 1.0f;
  if (max_norm <= 0.f) coef = 1.0f;
  return inv * coef;
}

// the reference updates the EMA every iteration, also when GradScaler skipped the optimizer step
__device__ __forceinline__ void ema_skipped_step(const float* __restrict__ p, float* __restrict__ ema, int64_t n, float ema_momentum) {
  if (ema != nullptr)
    for (int64_t i = (int64_t)blockIdx.x * ONT + threadIdx.x; i < n; i += (int64_t)gridDim.x * ONT)
      ema[i] = fmaf(ema[i], 1.0f - ema_momentum, ema_momentum * p[i]);
}

// every block has read stats / step; the LAST block to finish updates the scalar state and clears the statistics
__device__ __forceinline__ void finish_step(float* stats, float* scale, float* step, bool skip, const float* s_tot, float growth, float backoff,
                                            int growth_interval) {
  __shared__ unsigned int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(reinterpret_cast<unsigned int*>(stats + 3), 1u);
    s_last = (done == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    if (skip) {
      scale[0] *= backoff;  // GradScaler.update: back off, reset the growth tracker
      scale[1] = 0.f;
    } else {
      step[0] += 1.0f;
      const float tr = scale[1] + 1.0f;
      if (tr >= (float)growth_interval) { scale[0] *= growth; scale[1] = 0.f; } else { scale[1] = tr; }
    }
    stats[0] = s_tot[0];  // left for inspection: squared gradient norm / non-finite count of the step just taken
    stats[1] = s_tot[1];
    *reinterpret_cast<unsigned int*>(stats + 3) = 0u;
    __threadfence();
  }
}

__global__ void __launch_bounds__(ONT) adamw_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                         const float* __restrict__ wd, int64_t n, const float* __restrict__ hp, float beta1, float beta2,
                                                         float eps, float max_norm, float* stats, float* scale, float* step, float growth,
                                                         float backoff, int growth_interval, float* __restrict__ ema, float ema_momentum,
                                                         const float* __restrict__ partials, int n_partials) {
  pdl_wait();
  pdl_trigger();
  __shared__ float s_tot[2];
  step_totals(partials, n_partials, s_tot);
  const float sumsq = s_tot[0];
  const bool skip = s_tot[1] > 0.f;  // GradScaler.step: no optimizer step when any gradient is inf / nan
  const float lr = hp[0];
  if (skip) {
    ema_skipped_step(p, ema, n, ema_momentum);
  } else {
    const float gs = grad_scale(stats[2], sumsq, max_norm);
    const float t = step[0] + 1.0f;
    const float bc1 = 1.0f - powf(beta1, t), bc2 = 1.0f - powf(beta2, t);
    const float step_size = lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
    for (int64_t i = (int64_t)blockIdx.x * ONT + threadIdx.x; i < n; i += (int64_t)gridDim.x * ONT) {
      const float gi = g[i] * gs;
      float pi = p[i] * (1.0f - lr * wd[i]);
      const float mi = m[i] + (gi - m[i]) * (1.0f - beta1);  // exp_avg.lerp_(grad, 1 - beta1)
      const float vi = fmaf(v[i], beta2, (1.0f - beta2) * gi * gi);
      const float denom = sqrtf(vi) * inv_sqrt_bc2 + eps;
      pi -= step_size * (mi / denom);
      p[i] = pi;
      m[i] = mi;
      v[i] = vi;
      if (ema != nullptr) ema[i] = fmaf(ema[i], 1.0f - ema_momentum, ema_momentum * pi);
    }
  }
  finish_step(stats, scale, step, skip, s_tot, growth, backoff, growth_interval);
}

// torch.optim.SGD(momentum, dampening=0, nesterov, weight_decay) (the EfficientNet / MobileNet recipes: optim/sgd.py of the reference):
//   g' = g*unscale*clip + wd[i]*p;  buf = mu*buf + g' (a zero buffer makes the first step torch's buf = clone(g'));
//   p -= lr * (g' + mu*buf) with Nesterov, lr * buf without
__global__ void __launch_bounds__(ONT) sgd_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf,
                                                       const float* __restrict__ wd, int64_t n, const float* __restrict__ hp, float momentum,
                                                       int nesterov, float max_norm, float* stats, float* scale, float* step, float growth,
                                                       float backoff, int growth_interval, float* __restrict__ ema, float ema_momentum,
                                                       const float* __restrict__ partials, int n_partials) {
  pdl_wait();
  pdl_trigger();
  __shared__ float s_tot[2];
  step_totals(partials, n_partials, s_tot);
  const bool skip = s_tot[1] > 0.f;
  const float lr = hp[0];
  if (skip) {
    ema_skipped_step(p, ema, n, ema_momentum);
  } else {
    const float gs = grad_scale(stats[2], s_tot[0], max_norm);
    for (int64_t i = (int64_t)blockIdx.x * ONT + threadIdx.x; i < n; i += (int64_t)gridDim.x * ONT) {
      const float pi0 = p[i];
      const float gi = fmaf(wd[i], pi0, g[i] * gs);
      const float bi = fmaf(momentum, buf[i], gi);
      const float d = nesterov ? fmaf(momentum, bi, gi) : bi;
      const float pi = fmaf(-lr, d, pi0);
      p[i] = pi;
      buf[i] = bi;
      if (ema != nullptr) ema[i] = fmaf(ema[i], 1.0f - ema_momentum, ema_momentum * pi);
    }
  }
  finish_step(stats, scale, step, skip, s_tot, growth, backoff, growth_interval);
}

}  // namespace

extern "C" int cvb_grad_norm_blocks(int64_t n) {
  int blocks = (int)((n / 4 + ONT - 1) / ONT);
  const int cap = 4 * cvb_num_sms();
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return blocks;
}

extern "C" int cvb_grad_norm(const float* grads, int64_t n, const float* scale, float grad_div, float* stats, float* partials, cvb_stream_t stream) {
  CVB_CHECK(grads && scale && stats && partials && n > 0 && grad_div > 0.f && cvb_aligned16(grads), "cvb_grad_norm: bad arguments");
  CVB_CUDA(cvb_launch(grad_norm_kernel, cvb_grad_norm_blocks(n), ONT, 0, static_cast<cudaStream_t>(stream), grads, n, scale, grad_div, stats, partials));
  return 0;
}

extern "C" int cvb_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const float* weight_decay, int64_t n,
                              const float* hp, float beta1, float beta2, float eps, float max_norm, float* stats, float* scale, float* step,
                              float growth_factor, float backoff_factor, int growth_interval, float* ema, float ema_momentum, const float* partials,
                              cvb_stream_t stream) {
  CVB_CHECK(params && grads && exp_avg && exp_avg_sq && weight_decay && hp && stats && scale && step && partials && n > 0, "cvb_adamw_step: bad arguments");
  int blocks = (int)((n + ONT - 1) / ONT);
  const int cap = 8 * cvb_num_sms();
  if (blocks > cap) blocks = cap;
  CVB_CUDA(cvb_launch(adamw_step_kernel, blocks, ONT, 0, static_cast<cudaStream_t>(stream), params, grads, exp_avg, exp_avg_sq, weight_decay, n, hp, beta1,
                      beta2, eps, max_norm, stats, scale, step, growth_factor, backoff_factor, growth_interval, ema, ema_momentum, partials,
                      cvb_grad_norm_blocks(n)));
  return 0;
}

extern "C" int cvb_sgd_step(float* params, const float* grads, float* momentum_buf, const float* weight_decay, int64_t n, const float* hp, float momentum,
                            int nesterov, float max_norm, float* stats, float* scale, float* step, float growth_factor, float backoff_factor,
                            int growth_interval, float* ema, float ema_momentum, const float* partials, cvb_stream_t stream) {
  CVB_CHECK(params && grads && momentum_buf && weight_decay && hp && stats && scale && step && partials && n > 0, "cvb_sgd_step: bad arguments");
  CVB_CHECK(!nesterov || momentum > 0.f, "cvb_sgd_step: Nesterov momentum requires momentum > 0");
  int blocks = (int)((n + ONT - 1) / ONT);
  const int cap = 8 * cvb_num_sms();
  if (blocks > cap) blocks = cap;
  CVB_CUDA(cvb_launch(sgd_step_kernel, blocks, ONT, 0, static_cast<cudaStream_t>(stream), params, grads, momentum_buf, weight_decay, n, hp, momentum,
                      nesterov, max_norm, stats, scale, step, growth_factor, backoff_factor, growth_interval, ema, ema_momentum, partials,
                      cvb_grad_norm_blocks(n)));
  return 0;
}
