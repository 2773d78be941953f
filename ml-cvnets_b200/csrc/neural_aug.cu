// RangeAugment (arXiv 2212.10553) with learned brightness / contrast / noise ranges, and the stem's input gradient, sm_90a.
// Reference: cvnets/neural_augmentor/neural_aug.py (DistributionNeuralAugmentor), utils/neural_aug_utils.py, loss_fn/neural_augmentation.py.
//
// Every augmentation is affine per (sample, channel), so the shuffled chain collapses to  x_out = A x_mix + Bc + C eps  per (b, c):
//   brightness m:  (A, Bc, C) *= m
//   contrast   m:  mean = A mu_x + Bc + C mu_eps (the spatial mean of the CURRENT tensor);  A *= m;  Bc = (1 - m) mean + m Bc;  C *= m
//   noise      s:  C += s
// then x_aug = clip(x_out, 0, 1).  m = low + u (high - low), low / high = sigmoid(raw) (max - min) + min (the reference's Clip).
//
// Random draws (the order of the augmentations, each one's max(1, B / 2)-sample subset, the per-sample u, the N(0, 1) field eps) are counter
// hashes of the step's 64-bit key (cvb_rng_next): the forward, the backward and the tests recompute them; only the [4 + 3 B] draw table
// is stored.  All reductions are fp64 in a fixed order (one CTA per image plane, or one CTA in all): a step is bitwise reproducible.
#include "common.cuh"

namespace {

constexpr int NA_NT = 256;
constexpr int NA_PLAN_NT = 1024;
constexpr int NA_MAX_B = 4096;

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// independent sub-streams of one key
enum : uint64_t { S_ORDER = 0x5A17ull, S_SEL = 0x5E1Eull, S_U = 0x0C0Dull, S_EPS = 0xE95Bull };
__device__ __forceinline__ uint64_t sub_key(uint64_t key, uint64_t stream) { return mix64(key ^ mix64(stream)); }
__device__ __forceinline__ float u24(uint64_t r) { return (float)(r >> 40) * (1.0f / 16777216.0f); }  // [0, 1)

// eps[e] ~ N(0, 1), Box-Muller on one 64-bit hash (u1 in (0, 1]: |eps| <= 5.8)
__device__ __forceinline__ float na_eps(uint64_t ekey, int64_t e) {
  const uint64_t r = mix64(ekey + (uint64_t)e);
  const float u1 = (float)((r >> 40) + 1) * (1.0f / 16777216.0f);
  const float u2 = (float)(r & 0xFFFFFFu) * (1.0f / 16777216.0f);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

struct Mix {
  int mode;
  float lam;
  int x1, y1, x2, y2;
};
__device__ __forceinline__ Mix load_mix(const float* mix) {
  Mix m{0, 1.f, 0, 0, 0, 0};
  if (mix) {
    m.mode = (int)mix[0];
    m.lam = mix[1];
    m.x1 = (int)mix[2], m.y1 = (int)mix[3], m.x2 = (int)mix[4], m.y2 = (int)mix[5];
  }
  return m;
}
// x_mix of plane (b, c) at pixel i: the rule of cvb_stem_im2col (image.roll(1, 0) partner, fp32)
__device__ __forceinline__ float mixed(const float* __restrict__ X, const Mix& m, int B, int b, int c, int H, int W, int i) {
  const int64_t HW = (int64_t)H * W;
  float v = __ldg(X + ((int64_t)b * 3 + c) * HW + i);
  if (m.mode != 0) {
    const int bp = b == 0 ? B - 1 : b - 1;
    const float* P = X + ((int64_t)bp * 3 + c) * HW + i;
    if (m.mode == 1) {
      v = fmaf(m.lam, v, (1.0f - m.lam) * __ldg(P));
    } else {
      const int h = i / W, w = i - h * W;
      if (h >= m.y1 && h < m.y2 && w >= m.x1 && w < m.x2) v = __ldg(P);
    }
  }
  return v;
}

template <int N>
__device__ __forceinline__ void block_sum(double* v, double (*sm)[N]) {  // sm: [NA_NT / 32][N]; result in thread 0
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < N; ++k) sm[wid][k] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < N; ++k) {
      double s = 0.0;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += sm[w][k];
      v[k] = s;
    }
  }
}

// sampler parameters: raw (_low, _high) of brightness, contrast, noise (nullptr = augmentation disabled); bounds of the reference's Clips
struct NaParams {
  const float* raw[6];
};
struct NaGrads {
  float* raw[6];
};
__constant__ float c_lo_min[3] = {0.1f, 0.1f, 0.0f}, c_lo_max[3] = {0.9f, 0.9f, 0.00005f};
__constant__ float c_hi_min[3] = {1.1f, 1.1f, 0.0001f}, c_hi_max[3] = {10.0f, 10.0f, 1.0f};
__device__ __forceinline__ float sig(float r) { return 1.0f / (1.0f + expf(-r)); }

// draw table: tab[0..2] = augmentation index at each position of the order (-1 past the enabled ones), tab[3] = count,
// tab[4 + k B + b] = u of sample b for augmentation k if selected, else -1
__global__ void __launch_bounds__(NA_PLAN_NT) na_plan_kernel(const unsigned long long* __restrict__ key_ptr, int B, int n, int enabled,
                                                             float* __restrict__ tab) {
  __shared__ uint64_t hs[NA_MAX_B];
  pdl_wait();
  pdl_trigger();
  const uint64_t key = key_ptr[0];
  if (threadIdx.x == 0) {
    const uint64_t ko = sub_key(key, S_ORDER);
    int cnt = 0;
    int pos[3];
    for (int k = 0; k < 3; ++k) {
      pos[k] = -1;
      if (!(enabled >> k & 1)) continue;
      ++cnt;
      int r = 0;
      const uint64_t hk = mix64(ko + k);
      for (int j = 0; j < 3; ++j)
        if (j != k && (enabled >> j & 1)) {
          const uint64_t hj = mix64(ko + j);
          r += (hj < hk) || (hj == hk && j < k);
        }
      pos[k] = r;
    }
    for (int p = 0; p < 3; ++p) tab[p] = -1.f;
    for (int k = 0; k < 3; ++k)
      if (pos[k] >= 0) tab[pos[k]] = (float)k;
    tab[3] = (float)cnt;
  }
  for (int k = 0; k < 3; ++k) {
    float* row = tab + 4 + (int64_t)k * B;
    if (!(enabled >> k & 1)) {
      for (int b = threadIdx.x; b < B; b += NA_PLAN_NT) row[b] = -1.f;
      continue;
    }
    // a uniformly random n-subset: the n samples of smallest hash (ties broken by index)
    const uint64_t ks = sub_key(key, S_SEL + 16 * k), ku = sub_key(key, S_U + 16 * k);
    __syncthreads();
    for (int b = threadIdx.x; b < B; b += NA_PLAN_NT) hs[b] = mix64(ks + b);
    __syncthreads();
    for (int b = threadIdx.x; b < B; b += NA_PLAN_NT) {
      const uint64_t h = hs[b];
      int r = 0;
      for (int j = 0; j < B; ++j) {
        const uint64_t hj = hs[j];
        r += (hj < h) || (hj == h && j < b);
      }
      row[b] = r < n ? u24(mix64(ku + b)) : -1.f;
    }
  }
}

__global__ void __launch_bounds__(NA_NT) na_noise_kernel(const unsigned long long* __restrict__ key_ptr, int64_t total, float* __restrict__ eps) {
  pdl_wait();
  pdl_trigger();
  const uint64_t ke = sub_key(key_ptr[0], S_EPS);
  for (int64_t e = (int64_t)blockIdx.x * NA_NT + threadIdx.x; e < total; e += (int64_t)gridDim.x * NA_NT) eps[e] = na_eps(ke, e);
}

// one CTA per plane (b, c): mu_x = mean(x_mix), mu_e = mean(eps)
__global__ void __launch_bounds__(NA_NT) na_stats_kernel(const float* __restrict__ X, const float* __restrict__ mix,
                                                         const unsigned long long* __restrict__ key_ptr, int B, int H, int W, int need_eps,
                                                         double* __restrict__ mu_x, double* __restrict__ mu_e) {
  __shared__ double sm[NA_NT / 32][2];
  pdl_wait();
  pdl_trigger();
  const int plane = blockIdx.x, b = plane / 3, c = plane % 3;
  const int HW = H * W;
  const Mix m = load_mix(mix);
  const uint64_t ke = sub_key(key_ptr[0], S_EPS);
  double v[2] = {0.0, 0.0};
  for (int i = threadIdx.x; i < HW; i += NA_NT) {
    v[0] += mixed(X, m, B, b, c, H, W, i);
    if (need_eps) v[1] += na_eps(ke, (int64_t)plane * HW + i);
  }
  block_sum<2>(v, sm);
  if (threadIdx.x == 0) {
    mu_x[plane] = v[0] / HW;
    mu_e[plane] = v[1] / HW;
  }
}

// (A, Bc, C) of plane p after the chain, optionally keeping the state before each position and the magnitude used there
struct Chain {
  float A[4], Bc[4], C[4], m[3];
  int k[3];
};
__device__ __forceinline__ void bounds(const NaParams& P, int k, float& lo, float& hi) {
  lo = sig(*P.raw[2 * k]) * (c_lo_max[k] - c_lo_min[k]) + c_lo_min[k];
  hi = sig(*P.raw[2 * k + 1]) * (c_hi_max[k] - c_hi_min[k]) + c_hi_min[k];
}
__device__ __forceinline__ int run_chain(const float* __restrict__ tab, int B, int b, float mx, float me, const NaParams& P, Chain& ch) {
  const int cnt = (int)tab[3];
  ch.A[0] = 1.f, ch.Bc[0] = 0.f, ch.C[0] = 0.f;
  for (int s = 0; s < cnt; ++s) {
    const int k = (int)tab[s];
    const float u = tab[4 + (int64_t)k * B + b];
    float A = ch.A[s], Bc = ch.Bc[s], C = ch.C[s], mag = 0.f;
    ch.k[s] = k;
    if (u >= 0.f) {
      float lo, hi;
      bounds(P, k, lo, hi);
      mag = lo + u * (hi - lo);
      if (k == 0) {
        A *= mag, Bc *= mag, C *= mag;
      } else if (k == 1) {
        const float mean = A * mx + Bc + C * me;
        A *= mag, C *= mag;
        Bc = (1.f - mag) * mean + mag * Bc;
      } else {
        C += mag;
      }
    } else {
      ch.k[s] = -1;  // sample not selected for this augmentation
    }
    ch.m[s] = mag;
    ch.A[s + 1] = A, ch.Bc[s + 1] = Bc, ch.C[s + 1] = C;
  }
  return cnt;
}

__global__ void __launch_bounds__(NA_NT) na_compose_kernel(const float* __restrict__ tab, const double* __restrict__ mu_x, const double* __restrict__ mu_e,
                                                           const NaParams P, int B, float* __restrict__ coef) {
  pdl_wait();
  pdl_trigger();
  for (int p = blockIdx.x * NA_NT + threadIdx.x; p < 3 * B; p += gridDim.x * NA_NT) {
    Chain ch;
    const int cnt = run_chain(tab, B, p / 3, (float)mu_x[p], (float)mu_e[p], P, ch);
    coef[3 * p] = ch.A[cnt], coef[3 * p + 1] = ch.Bc[cnt], coef[3 * p + 2] = ch.C[cnt];
  }
}

// one CTA per plane: Y = clip(A x_mix + Bc + C eps, 0, 1);  sq[plane] = sum (Y - x_mix)^2
__global__ void __launch_bounds__(NA_NT) na_apply_kernel(const float* __restrict__ X, const float* __restrict__ mix,
                                                         const unsigned long long* __restrict__ key_ptr, const float* __restrict__ coef, int B, int H,
                                                         int W, int need_eps, float* __restrict__ Y, double* __restrict__ sq) {
  __shared__ double sm[NA_NT / 32][1];
  pdl_wait();
  pdl_trigger();
  const int plane = blockIdx.x, b = plane / 3, c = plane % 3;
  const int HW = H * W;
  const Mix m = load_mix(mix);
  const uint64_t ke = sub_key(key_ptr[0], S_EPS);
  const float A = coef[3 * plane], Bc = coef[3 * plane + 1], C = coef[3 * plane + 2];
  float* y = Y + (int64_t)plane * HW;
  double v[1] = {0.0};
  for (int i = threadIdx.x; i < HW; i += NA_NT) {
    const float xm = mixed(X, m, B, b, c, H, W, i);
    float o = fmaf(A, xm, Bc);
    if (need_eps) o = fmaf(C, na_eps(ke, (int64_t)plane * HW + i), o);
    o = fminf(fmaxf(o, 0.f), 1.f);
    y[i] = o;
    const float d = o - xm;
    v[0] += (double)(d * d);
  }
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) sq[plane] = v[0];
}

// one CTA per plane: g = [0 <= pre <= 1] (dY + 2 g_sq (Y - x_mix));  red[plane] = (sum g x_mix, sum g, sum g eps)
__global__ void __launch_bounds__(NA_NT) na_bwd_reduce_kernel(const float* __restrict__ DY, const double* __restrict__ g_sq, const float* __restrict__ X,
                                                              const float* __restrict__ mix, const unsigned long long* __restrict__ key_ptr,
                                                              const float* __restrict__ coef, int B, int H, int W, int need_eps,
                                                              double* __restrict__ red) {
  __shared__ double sm[NA_NT / 32][3];
  pdl_wait();
  pdl_trigger();
  const int plane = blockIdx.x, b = plane / 3, c = plane % 3;
  const int HW = H * W;
  const Mix m = load_mix(mix);
  const uint64_t ke = sub_key(key_ptr[0], S_EPS);
  const float A = coef[3 * plane], Bc = coef[3 * plane + 1], C = coef[3 * plane + 2];
  const float gs2 = g_sq ? (float)(2.0 * g_sq[plane]) : 0.f;
  const float* dy = DY ? DY + (int64_t)plane * HW : nullptr;
  double v[3] = {0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < HW; i += NA_NT) {
    const float xm = mixed(X, m, B, b, c, H, W, i);
    const float e = need_eps ? na_eps(ke, (int64_t)plane * HW + i) : 0.f;
    const float pre = fmaf(C, e, fmaf(A, xm, Bc));
    if (pre < 0.f || pre > 1.f) continue;  // torch.clamp passes the gradient where min <= x <= max
    float g = dy ? __ldg(dy + i) : 0.f;
    g = fmaf(gs2, pre - xm, g);
    v[0] += (double)(g * xm);
    v[1] += (double)g;
    v[2] += (double)(g * e);
  }
  block_sum<3>(v, sm);
  if (threadIdx.x == 0) red[3 * plane] = v[0], red[3 * plane + 1] = v[1], red[3 * plane + 2] = v[2];
}

// one CTA: chain rule of the per-plane sums through the composition, the draws and the sigmoid clips; grads[j] = d loss / d raw[j]
__global__ void __launch_bounds__(NA_NT) na_param_grad_kernel(const float* __restrict__ tab, const double* __restrict__ mu_x,
                                                              const double* __restrict__ mu_e, const double* __restrict__ red, const NaParams P, int B,
                                                              NaGrads G) {
  __shared__ double sm[NA_NT / 32][6];
  pdl_wait();
  pdl_trigger();
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // (d low, d high) per augmentation
  for (int p = threadIdx.x; p < 3 * B; p += NA_NT) {
    const int b = p / 3;
    const float mx = (float)mu_x[p], me = (float)mu_e[p];
    Chain ch;
    const int cnt = run_chain(tab, B, b, mx, me, P, ch);
    float a = (float)red[3 * p], bb = (float)red[3 * p + 1], cc = (float)red[3 * p + 2];
    for (int s = cnt - 1; s >= 0; --s) {
      const int k = ch.k[s];
      if (k < 0) continue;
      const float A = ch.A[s], Bc = ch.Bc[s], C = ch.C[s], mag = ch.m[s];
      float dm;
      if (k == 0) {
        dm = a * A + bb * Bc + cc * C;
        a *= mag, bb *= mag, cc *= mag;
      } else if (k == 1) {
        const float mean = A * mx + Bc + C * me;
        dm = a * A + bb * (Bc - mean) + cc * C;
        a = a * mag + bb * (1.f - mag) * mx;
        cc = cc * mag + bb * (1.f - mag) * me;
      } else {
        dm = cc;
      }
      const float u = tab[4 + (int64_t)k * B + b];
      acc[2 * k] += (double)(dm * (1.f - u));
      acc[2 * k + 1] += (double)(dm * u);
    }
  }
  block_sum<6>(acc, sm);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 3; ++k) {
      if (!P.raw[2 * k]) continue;
      const float sl = sig(*P.raw[2 * k]), sh = sig(*P.raw[2 * k + 1]);
      *G.raw[2 * k] = (float)acc[2 * k] * sl * (1.f - sl) * (c_lo_max[k] - c_lo_min[k]);
      *G.raw[2 * k + 1] = (float)acc[2 * k + 1] * sh * (1.f - sh) * (c_hi_max[k] - c_hi_min[k]);
    }
  }
}

// loss_fn/neural_augmentation.py:_forward_psnr:  L = alpha / 65025 * mean_b smooth_l1(mse_b - t[step]),  mse_b = 65025 sum_c sq[b, c] / (3 H W)
__device__ __forceinline__ float na_target(const float* __restrict__ target, int T, const long long* __restrict__ step) {
  long long s = step ? step[0] : 0;
  if (s >= T || s < 0) s = T - 1;
  return target[s];
}
__global__ void __launch_bounds__(NA_NT) na_loss_fwd_kernel(const double* __restrict__ sq, int B, double inv_chw, const float* __restrict__ target, int T,
                                                            const long long* __restrict__ step, float alpha, float w_na, const float* __restrict__ ce,
                                                            float w_ce, float* __restrict__ loss, float* __restrict__ parts) {
  __shared__ double sm[NA_NT / 32][1];
  pdl_wait();
  pdl_trigger();
  const float t = na_target(target, T, step);
  double v[1] = {0.0};
  for (int b = threadIdx.x; b < B; b += NA_NT) {
    const float mse = (float)((sq[3 * b] + sq[3 * b + 1] + sq[3 * b + 2]) * 65025.0 * inv_chw);
    const float d = mse - t, ad = fabsf(d);
    v[0] += (double)(ad < 1.f ? 0.5f * d * d : ad - 0.5f);
  }
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) {
    const float na = (float)(v[0] / B) * (alpha / 65025.0f);
    const float c = ce ? ce[0] : 0.f;
    loss[0] = fmaf(w_na, na, ce ? w_ce * c : 0.f);
    if (parts) parts[0] = c, parts[1] = na;
  }
}

__global__ void __launch_bounds__(NA_NT) na_loss_bwd_kernel(const double* __restrict__ sq, int B, double inv_chw, const float* __restrict__ target, int T,
                                                            const long long* __restrict__ step, float alpha, float w_na, const float* __restrict__ grad_out,
                                                            const float* __restrict__ grad_scale, double* __restrict__ g_sq, float* __restrict__ g_ce,
                                                            float w_ce) {
  pdl_wait();
  pdl_trigger();
  const float t = na_target(target, T, step);
  const float go = grad_out ? grad_out[0] : 1.f;
  const float gs = go * (grad_scale ? grad_scale[0] : 1.f) * w_na;
  if (g_ce && blockIdx.x == 0 && threadIdx.x == 0) g_ce[0] = go * w_ce;  // the cross entropy's backward applies the loss scale itself
  for (int b = blockIdx.x * NA_NT + threadIdx.x; b < B; b += gridDim.x * NA_NT) {
    const float mse = (float)((sq[3 * b] + sq[3 * b + 1] + sq[3 * b + 2]) * 65025.0 * inv_chw);
    const float d = fminf(fmaxf(mse - t, -1.f), 1.f);
    const double g = (double)(gs * (alpha / 65025.0f) / B * d) * 65025.0 * inv_chw;
    g_sq[3 * b] = g_sq[3 * b + 1] = g_sq[3 * b + 2] = g;
  }
}

// Stem input gradient: dX[b, ci, h, w] = sum over (co, u, v) of dy[b, oh, ow, co] W[co, ci, u, v], h = 2 oh + u - 1, w = 2 ow + v - 1,
// dy = bf16(p0 dz + p1 y + p2) (the BatchNorm-backward load mode the weight gradient applies).  One thread per 2 x 2 input block
// (2i..2i+1, 2j..2j+1): it reads the four output pixels (i..i+1, j..j+1) once, in 8-channel chunks.
__global__ void __launch_bounds__(NA_NT) stem_dgrad_kernel(const bf16* __restrict__ DZ, const bf16* __restrict__ Yp, const float* __restrict__ coef,
                                                           const bf16* __restrict__ Wp, int B, int Ho, int Wo, int C0, float* __restrict__ DX) {
  __shared__ float wsm[27][64];  // [ci*9 + u*3 + v][co]
  __shared__ float cs[3][64];
  pdl_wait();
  pdl_trigger();
  for (int t = threadIdx.x; t < 27 * C0; t += NA_NT) wsm[t % 27][t / 27] = __bfloat162float(Wp[(t / 27) * 32 + t % 27]);
  for (int t = threadIdx.x; t < 3 * C0; t += NA_NT) cs[t / C0][t % C0] = coef[t];
  __syncthreads();
  const int H = 2 * Ho, W = 2 * Wo;
  const int64_t total = (int64_t)B * Ho * Wo;
  for (int64_t idx = (int64_t)blockIdx.x * NA_NT + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * NA_NT) {
    const int j = (int)(idx % Wo), i = (int)((idx / Wo) % Ho);
    const int b = (int)(idx / ((int64_t)Wo * Ho));
    float acc[3][2][2];
#pragma unroll
    for (int ci = 0; ci < 3; ++ci)
#pragma unroll
      for (int dh = 0; dh < 2; ++dh) acc[ci][dh][0] = acc[ci][dh][1] = 0.f;
    for (int c8 = 0; c8 < C0; c8 += 8) {
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        if (i + a >= Ho) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          if (j + e >= Wo) continue;
          const int64_t row = ((int64_t)b * Ho + i + a) * Wo + j + e;
          float dz[8], yy[8];
          unpack8(ldg16(DZ + row * C0 + c8), dz);
          unpack8(ldg16(Yp + row * C0 + c8), yy);
#pragma unroll
          for (int q = 0; q < 8; ++q) dz[q] = bf16_round(fmaf(cs[0][c8 + q], dz[q], fmaf(cs[1][c8 + q], yy[q], cs[2][c8 + q])));
          // input rows fed by output row i + a: a = 0 -> (dh 0, u 1), (dh 1, u 2);  a = 1 -> (dh 1, u 0).  Columns alike.
#pragma unroll
          for (int dh = 0; dh < 2; ++dh) {
            if (a == 1 && dh == 0) continue;
            const int u = dh == 0 ? 1 : (a == 0 ? 2 : 0);
#pragma unroll
            for (int dw = 0; dw < 2; ++dw) {
              if (e == 1 && dw == 0) continue;
              const int v = dw == 0 ? 1 : (e == 0 ? 2 : 0);
#pragma unroll
              for (int ci = 0; ci < 3; ++ci) {
                const float* wr = &wsm[ci * 9 + u * 3 + v][c8];
                float s = acc[ci][dh][dw];
#pragma unroll
                for (int q = 0; q < 8; ++q) s = fmaf(dz[q], wr[q], s);
                acc[ci][dh][dw] = s;
              }
            }
          }
        }
      }
    }
#pragma unroll
    for (int ci = 0; ci < 3; ++ci)
#pragma unroll
      for (int dh = 0; dh < 2; ++dh)
        *reinterpret_cast<float2*>(DX + (((int64_t)b * 3 + ci) * H + 2 * i + dh) * W + 2 * j) = make_float2(acc[ci][dh][0], acc[ci][dh][1]);
  }
}

// ViT / CLIP conv-stem input gradient (3 -> C0, k = stride = 4, pad 1): dX[b, ci, 4i-1+u, 4j-1+v] = sum over co of dy[b, i, j, co] W[co, (4u+v)*3 + ci],
// dy = bf16(p0 dz + p1 y + p2).  Stride = kernel, so the windows never overlap and every dX element has exactly one writer (no atomics, no
// memset, bitwise reproducible).  The padding shifts the windows by one pixel: window i covers rows 4i-1 .. 4i+2, so image row / column -1 is
// padding and H-1 / W-1 lie in no window (gradient 0).  The aligned float4 dX[.., 4q .. 4q+3] therefore holds columns v = 1..3 of patch q and
// v = 0 of patch q+1.  A warp owns 15 consecutive patches of one patch row and also computes the 16th (the right neighbour; zero past the
// row's end, which yields the W-1 column), stages the [16 x 48] result in shared memory and writes each image row as float4s, neighbouring
// patches on neighbouring lanes.  The [16 x C0] x [C0 x 48] product runs on mma.sync m16n8k16 with the weight resident in shared memory; the
// reduction order over channels is permuted so that each lane reads 8 consecutive channels (16 bytes) of its two rows per 32-channel step.
constexpr int PS_NT = 384;
constexpr int PS_WARPS = PS_NT / 32;
constexpr int PS_OWN = 15;    // patches a warp writes; it computes PS_OWN + 1
constexpr int PS_LDS = 56;    // staging row stride (floats): conflict-free float2 stores of the accumulator fragments
constexpr int PS_MAX_C0 = 320;

__host__ __device__ constexpr int ps_ldw(int C0) { return C0 + ((32 - C0 % 64) + 64) % 64; }  // weight row stride (bf16) = 32 mod 64
__host__ __device__ constexpr size_t ps_smem(int C0) {
  return (size_t)48 * ps_ldw(C0) * 2 + (size_t)3 * C0 * 4 + (size_t)PS_WARPS * 16 * PS_LDS * 4;
}

// n bf16 BatchNorm-backward values of one row (n = 8 or 4): channels c .. c+n-1, zero for a row past the patch row's end
template <int N>
__device__ __forceinline__ void ps_bnb(const uint32_t* z, const uint32_t* y, const float* cs, int C0, int c, bool valid, uint32_t* d) {
#pragma unroll
  for (int q = 0; q < N / 2; ++q) {
    const float2 zz = unpack_bf162(z[q]), yy = unpack_bf162(y[q]);
    const int k = c + 2 * q;
    const float lo = fmaf(cs[k], zz.x, fmaf(cs[C0 + k], yy.x, cs[2 * C0 + k]));
    const float hi = fmaf(cs[k + 1], zz.y, fmaf(cs[C0 + k + 1], yy.y, cs[2 * C0 + k + 1]));
    d[q] = valid ? pack_bf162(lo, hi) : 0u;
  }
}

__global__ void __launch_bounds__(PS_NT) patch_stem_dgrad_kernel(const bf16* __restrict__ DZ, const bf16* __restrict__ Yp, const float* __restrict__ coef,
                                                                 const bf16* __restrict__ Wp, int B, int Ho, int Wo, int C0, float* __restrict__ DX) {
  extern __shared__ __align__(16) unsigned char ps_raw[];
  const int ldw = ps_ldw(C0);
  bf16* sW = reinterpret_cast<bf16*>(ps_raw);                          // [48][ldw]: column n of the prepared [C0, 48] weight, channels contiguous
  float* cs = reinterpret_cast<float*>(ps_raw + (size_t)48 * ldw * 2);  // [3][C0]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  float* stg = cs + 3 * C0 + warp * 16 * PS_LDS;                        // [16][PS_LDS] per warp
  pdl_wait();
  pdl_trigger();
  for (int t = threadIdx.x; t < 48 * C0; t += PS_NT) sW[(t % 48) * ldw + t / 48] = Wp[t];
  for (int t = threadIdx.x; t < 3 * C0; t += PS_NT) cs[t] = coef[t];
  __syncthreads();
  const int H = 4 * Ho, W = 4 * Wo;
  const int nchunk = (Wo + PS_OWN - 1) / PS_OWN;
  const int64_t tiles = (int64_t)B * Ho * nchunk;
  const int nfull = C0 / 32;
  const bool tail = (C0 % 32) != 0;
  for (int64_t t = (int64_t)blockIdx.x * PS_WARPS + warp; t < tiles; t += (int64_t)gridDim.x * PS_WARPS) {
    const int64_t prow = t / nchunk;  // b * Ho + i
    const int j0 = (int)(t % nchunk) * PS_OWN;
    const bool v_lo = j0 + g < Wo, v_hi = j0 + g + 8 < Wo;
    const bf16* zlo = DZ + (prow * Wo + j0 + g) * C0;
    const bf16* ylo = Yp + (prow * Wo + j0 + g) * C0;
    const bf16* zhi = zlo + 8 * (int64_t)C0;
    const bf16* yhi = ylo + 8 * (int64_t)C0;
    float acc[6][4];
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
    const uint4 zero4 = make_uint4(0, 0, 0, 0);
    uint4 nz0 = zero4, ny0 = zero4, nz1 = zero4, ny1 = zero4;
    if (nfull > 0) {
      const int c = 8 * tq;
      if (v_lo) nz0 = ldg16_stream(zlo + c), ny0 = ldg16_stream(ylo + c);
      if (v_hi) nz1 = ldg16_stream(zhi + c), ny1 = ldg16_stream(yhi + c);
    }
    for (int s = 0; s < nfull; ++s) {
      const uint4 z0 = nz0, y0 = ny0, z1 = nz1, y1 = ny1;
      if (s + 1 < nfull) {  // the next 32 channels are in flight while these go through the tensor cores
        const int c = 32 * (s + 1) + 8 * tq;
        if (v_lo) nz0 = ldg16_stream(zlo + c), ny0 = ldg16_stream(ylo + c);
        if (v_hi) nz1 = ldg16_stream(zhi + c), ny1 = ldg16_stream(yhi + c);
      }
      const int c = 32 * s + 8 * tq;
      uint32_t dl[4], dh[4];
      ps_bnb<8>(&z0.x, &y0.x, cs, C0, c, v_lo, dl);
      ps_bnb<8>(&z1.x, &y1.x, cs, C0, c, v_hi, dh);
      const uint32_t a0[4] = {dl[0], dh[0], dl[1], dh[1]};  // channels c+0..3: k-step 2s
      const uint32_t a1[4] = {dl[2], dh[2], dl[3], dh[3]};  // channels c+4..7: k-step 2s+1
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) {
        const uint4 w = *reinterpret_cast<const uint4*>(sW + (8 * nt + g) * ldw + c);
        mma_bf16_16816(acc[nt], a0, w.x, w.y);
        mma_bf16_16816(acc[nt], a1, w.z, w.w);
      }
    }
    if (tail) {  // C0 = 32 nfull + 16: one k-step, 4 channels (8 bytes) per lane and row
      const int c = 32 * nfull + 4 * tq;
      uint2 z0 = make_uint2(0, 0), y0 = z0, z1 = z0, y1 = z0;
      if (v_lo) z0 = __ldg(reinterpret_cast<const uint2*>(zlo + c)), y0 = __ldg(reinterpret_cast<const uint2*>(ylo + c));
      if (v_hi) z1 = __ldg(reinterpret_cast<const uint2*>(zhi + c)), y1 = __ldg(reinterpret_cast<const uint2*>(yhi + c));
      uint32_t dl[2], dh[2];
      ps_bnb<4>(&z0.x, &y0.x, cs, C0, c, v_lo, dl);
      ps_bnb<4>(&z1.x, &y1.x, cs, C0, c, v_hi, dh);
      const uint32_t a[4] = {dl[0], dh[0], dl[1], dh[1]};
#pragma unroll
      for (int nt = 0; nt < 6; ++nt) {
        const uint2 w = *reinterpret_cast<const uint2*>(sW + (8 * nt + g) * ldw + c);
        mma_bf16_16816(acc[nt], a, w.x, w.y);
      }
    }
#pragma unroll
    for (int nt = 0; nt < 6; ++nt) {
      *reinterpret_cast<float2*>(stg + g * PS_LDS + 8 * nt + 2 * tq) = make_float2(acc[nt][0], acc[nt][1]);
      *reinterpret_cast<float2*>(stg + (g + 8) * PS_LDS + 8 * nt + 2 * tq) = make_float2(acc[nt][2], acc[nt][3]);
    }
    __syncwarp();
    const int qo = lane & 15, half = lane >> 4;
    const int b = (int)(prow / Ho), i = (int)(prow % Ho);
    if (qo < PS_OWN && j0 + qo < Wo) {
      const float* p = stg + qo * PS_LDS;
      float* base = DX + (int64_t)b * 3 * H * W + 4 * (j0 + qo);
#pragma unroll
      for (int it = 0; it < 6; ++it) {
        const int combo = 2 * it + half, u = combo / 3, ci = combo % 3;
        const int r = 4 * i - 1 + u;
        if (r >= 0)
          *reinterpret_cast<float4*>(base + ((int64_t)ci * H + r) * W) =
              make_float4(p[(4 * u + 1) * 3 + ci], p[(4 * u + 2) * 3 + ci], p[(4 * u + 3) * 3 + ci], p[PS_LDS + (4 * u) * 3 + ci]);
      }
      if (i == Ho - 1)  // image row H-1 lies in no window
        for (int ci = half; ci < 3; ci += 2) *reinterpret_cast<float4*>(base + ((int64_t)ci * H + H - 1) * W) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();
  }
}

int grid_for(int64_t items) {
  int64_t g = (items + NA_NT - 1) / NA_NT;
  const int64_t cap = 8 * (int64_t)cvb_num_sms();
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

int params_of(const float* const* raw, NaParams* P, const char* who) {
  for (int k = 0; k < 3; ++k) {
    CVB_CHECK(!raw[2 * k] == !raw[2 * k + 1], "%s: augmentation %d needs both _low and _high (or neither)", who, k);
    P->raw[2 * k] = raw[2 * k], P->raw[2 * k + 1] = raw[2 * k + 1];
  }
  return 0;
}

}  // namespace

extern "C" int cvb_na_plan(const void* key, int B, int enabled, float* tab, cvb_stream_t stream) {
  CVB_CHECK(key && tab && B > 0 && B <= NA_MAX_B && enabled > 0 && enabled < 8, "cvb_na_plan: bad arguments (1 <= B <= %d, enabled in 1..7)", NA_MAX_B);
  const int n = B / 2 > 1 ? B / 2 : 1;
  CVB_CUDA(cvb_launch(na_plan_kernel, 1, NA_PLAN_NT, 0, static_cast<cudaStream_t>(stream), static_cast<const unsigned long long*>(key), B, n, enabled, tab));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_noise(const void* key, int B, int H, int W, float* eps, cvb_stream_t stream) {
  CVB_CHECK(key && eps && B > 0 && H > 0 && W > 0, "cvb_na_noise: bad arguments");
  const int64_t total = (int64_t)B * 3 * H * W;
  CVB_CUDA(cvb_launch(na_noise_kernel, grid_for(total), NA_NT, 0, static_cast<cudaStream_t>(stream), static_cast<const unsigned long long*>(key), total, eps));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_stats(const float* X, const float* mix, const void* key, int B, int H, int W, int need_eps, double* mu_x, double* mu_e,
                            cvb_stream_t stream) {
  CVB_CHECK(X && key && mu_x && mu_e && B > 0 && H > 0 && W > 0, "cvb_na_stats: bad arguments");
  CVB_CUDA(cvb_launch(na_stats_kernel, 3 * B, NA_NT, 0, static_cast<cudaStream_t>(stream), X, mix, static_cast<const unsigned long long*>(key), B, H, W,
                      need_eps, mu_x, mu_e));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_compose(const float* tab, const double* mu_x, const double* mu_e, const float* const* raw, int B, float* coef, cvb_stream_t stream) {
  NaParams P;
  CVB_CHECK(tab && mu_x && mu_e && raw && coef && B > 0, "cvb_na_compose: bad arguments");
  if (params_of(raw, &P, "cvb_na_compose")) return 1;
  CVB_CUDA(cvb_launch(na_compose_kernel, grid_for(3 * B), NA_NT, 0, static_cast<cudaStream_t>(stream), tab, mu_x, mu_e, P, B, coef));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_apply(const float* X, const float* mix, const void* key, const float* coef, int B, int H, int W, int need_eps, float* Y, double* sq,
                            cvb_stream_t stream) {
  CVB_CHECK(X && key && coef && Y && sq && B > 0 && H > 0 && W > 0, "cvb_na_apply: bad arguments");
  CVB_CUDA(cvb_launch(na_apply_kernel, 3 * B, NA_NT, 0, static_cast<cudaStream_t>(stream), X, mix, static_cast<const unsigned long long*>(key), coef, B, H, W,
                      need_eps, Y, sq));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_bwd_reduce(const float* DY, const double* g_sq, const float* X, const float* mix, const void* key, const float* coef, int B, int H, int W,
                                 int need_eps, double* red, cvb_stream_t stream) {
  CVB_CHECK(X && key && coef && red && B > 0 && H > 0 && W > 0, "cvb_na_bwd_reduce: bad arguments");
  CVB_CUDA(cvb_launch(na_bwd_reduce_kernel, 3 * B, NA_NT, 0, static_cast<cudaStream_t>(stream), DY, g_sq, X, mix, static_cast<const unsigned long long*>(key),
                      coef, B, H, W, need_eps, red));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_param_grad(const float* tab, const double* mu_x, const double* mu_e, const double* red, const float* const* raw, int B,
                                 float* const* grads, cvb_stream_t stream) {
  NaParams P;
  NaGrads G;
  CVB_CHECK(tab && mu_x && mu_e && red && raw && grads && B > 0, "cvb_na_param_grad: bad arguments");
  if (params_of(raw, &P, "cvb_na_param_grad")) return 1;
  for (int j = 0; j < 6; ++j) {
    CVB_CHECK(!P.raw[j] == !grads[j], "cvb_na_param_grad: gradient %d given without its parameter (or the reverse)", j);
    G.raw[j] = grads[j];
  }
  CVB_CUDA(cvb_launch(na_param_grad_kernel, 1, NA_NT, 0, static_cast<cudaStream_t>(stream), tab, mu_x, mu_e, red, P, B, G));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_loss_fwd(const double* sq, int B, int H, int W, const float* target, int T, const int64_t* step, float alpha, float w_na,
                               const float* ce, float w_ce, float* loss, float* parts, cvb_stream_t stream) {
  CVB_CHECK(sq && target && loss && B > 0 && H > 0 && W > 0 && T > 0, "cvb_na_loss_fwd: bad arguments");
  CVB_CUDA(cvb_launch(na_loss_fwd_kernel, 1, NA_NT, 0, static_cast<cudaStream_t>(stream), sq, B, 1.0 / (3.0 * H * W), target, T,
                      reinterpret_cast<const long long*>(step), alpha, w_na, ce, w_ce, loss, parts));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_na_loss_bwd(const double* sq, int B, int H, int W, const float* target, int T, const int64_t* step, float alpha, float w_na,
                               const float* grad_out, const float* grad_scale, double* g_sq, float* g_ce, float w_ce, cvb_stream_t stream) {
  CVB_CHECK(sq && target && g_sq && B > 0 && H > 0 && W > 0 && T > 0, "cvb_na_loss_bwd: bad arguments");
  CVB_CUDA(cvb_launch(na_loss_bwd_kernel, grid_for(B), NA_NT, 0, static_cast<cudaStream_t>(stream), sq, B, 1.0 / (3.0 * H * W), target, T,
                      reinterpret_cast<const long long*>(step), alpha, w_na, grad_out, grad_scale, g_sq, g_ce, w_ce));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_stem_dgrad(const void* dz, const void* y, const float* coef, const void* w, int B, int Ho, int Wo, int C0, float* dX, cvb_stream_t stream) {
  CVB_CHECK(dz && y && coef && w && dX && B > 0 && Ho > 0 && Wo > 0 && C0 > 0 && C0 <= 64 && C0 % 8 == 0,
            "cvb_stem_dgrad: bad arguments (C0 a multiple of 8 up to 64)");
  CVB_CHECK(cvb_aligned16(dz) && cvb_aligned16(y) && (reinterpret_cast<uintptr_t>(dX) & 7) == 0, "cvb_stem_dgrad: misaligned operand");
  CVB_CUDA(cvb_launch(stem_dgrad_kernel, grid_for((int64_t)B * Ho * Wo), NA_NT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(dz),
                      static_cast<const bf16*>(y), coef, static_cast<const bf16*>(w), B, Ho, Wo, C0, dX));
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_patch_stem_dgrad(const void* dz, const void* y, const float* coef, const void* w, int B, int Ho, int Wo, int C0, float* dX,
                                    cvb_stream_t stream) {
  CVB_CHECK(dz && y && coef && w && dX && B > 0 && Ho > 0 && Wo > 0 && C0 >= 16 && C0 <= PS_MAX_C0 && C0 % 16 == 0,
            "cvb_patch_stem_dgrad: bad arguments (C0 a multiple of 16 up to %d)", PS_MAX_C0);
  CVB_CHECK(cvb_aligned16(dz) && cvb_aligned16(y) && cvb_aligned16(dX) && cvb_aligned16(coef), "cvb_patch_stem_dgrad: misaligned operand");
  static bool attr = false;
  if (!attr) {
    CVB_CUDA(cudaFuncSetAttribute(patch_stem_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ps_smem(PS_MAX_C0)));
    attr = true;
  }
  const int64_t tiles = (int64_t)B * Ho * ((Wo + PS_OWN - 1) / PS_OWN);
  const int64_t want = (tiles + PS_WARPS - 1) / PS_WARPS;
  const int grid = (int)(want < cvb_num_sms() ? want : cvb_num_sms());  // persistent: at most one CTA per SM
  CVB_CUDA(cvb_launch(patch_stem_dgrad_kernel, grid, PS_NT, ps_smem(C0), static_cast<cudaStream_t>(stream), static_cast<const bf16*>(dz),
                      static_cast<const bf16*>(y), coef, static_cast<const bf16*>(w), B, Ho, Wo, C0, dX));
  CVB_LAUNCH_CHECK();
  return 0;
}
