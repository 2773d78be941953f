// BatchNorm / GroupNorm bookkeeping, materialisation, reductions, pooling, stem im2col and weight preparation (sm_90a).
// All tensor passes are 16-byte vectorised over the channel dimension of the [M, C] channels-last matrix; per-channel
// reductions keep a fixed channel chunk per thread (threads = multiple of C/8), reduce in smem, then one fp64 atomic per
// channel per CTA.
#include <stdarg.h>

#include "common.cuh"

// ---------------------------------------------------------------------------------------------- error / device plumbing
static thread_local char g_err[512] = "";
void cvb_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
extern "C" const char* cvb_last_error(void) { return g_err; }
extern "C" int cvb_abi_version(void) { return CVB_ABI_VERSION; }
static int g_pdl_enabled = 1;
int cvb_pdl_enabled() { return g_pdl_enabled; }
extern "C" int cvb_set_pdl_enabled(int on) {
  int old = g_pdl_enabled;
  g_pdl_enabled = on ? 1 : 0;
  return old;
}

int cvb_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}
__global__ void __launch_bounds__(256) det_add_kernel(const double* __restrict__ s, float* __restrict__ dst, int rows, int cols, int ld) {
  pdl_wait();
  pdl_trigger();
  const int64_t n = (int64_t)rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols), c = (int)(i % cols);
    dst[(size_t)r * ld + c] += (float)s[i];
  }
}
DetScratch::~DetScratch() {
  // an early return: the failure that caused it has set the message, so a failed free here only clears its pending error
  if (p_ && cudaFreeAsync(p_, st_) != cudaSuccess) (void)cudaGetLastError();
}
int DetScratch::alloc(size_t n) {
  static bool pool_set = false;
  if (!pool_set) {  // keep freed scratch in the device's default pool instead of returning it to the driver at every synchronisation
    int dev = 0;
    cudaMemPool_t pool;
    CVB_CUDA(cudaGetDevice(&dev));
    CVB_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
    uint64_t keep = UINT64_MAX;
    CVB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    pool_set = true;
  }
  CVB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&p_), n * sizeof(double), st_));
  CVB_CUDA(cudaMemsetAsync(p_, 0, n * sizeof(double), st_));
  return 0;
}
int DetScratch::add(size_t offset, float* dst, int rows, int cols, int ld) {
  const int64_t n = (int64_t)rows * cols;
  const int grid = (int)std::min<int64_t>((n + 255) / 256, 4 * (int64_t)cvb_num_sms());
  CVB_CUDA(cvb_launch(det_add_kernel, grid, 256, 0, st_, static_cast<const double*>(p_ + offset), dst, rows, cols, ld));
  return 0;
}
int DetScratch::release() {
  double* p = p_;
  p_ = nullptr;
  CVB_CUDA(cudaFreeAsync(p, st_));
  return 0;
}
extern "C" int cvb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  CVB_CUDA(cudaGetDevice(&dev));
  if (sm_count) CVB_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev));
  if (cc_major) CVB_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev));
  if (cc_minor) CVB_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
  return 0;
}

// ---------------------------------------------------------------------------------------------- TMA tensor maps (host)
typedef CUresult (*cvb_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                        const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// bf16 tiled tensor map of `rank` dimensions (innermost first), unit element strides, 128-byte L2 promotion, zero fill out of bounds
static int encode_bf16(CUtensorMap* map, cuuint32_t rank, const void* base, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                       CUtensorMapSwizzle swizzle) {
  static cvb_encode_tiled_fn enc = nullptr;
  if (!enc) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<cvb_encode_tiled_fn>(p);
  }
  CVB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  CVB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (%u-D) failed with %d", rank, (int)r);
  return 0;
}
int cvb_make_tmap_nhwc(CUtensorMap* map, const void* base, int B, int H, int W, int C, int boxH, int boxW, int boxC) {
  CVB_CHECK(boxC * 2 <= 128 && boxW <= 256 && boxH <= 256 && C % 8 == 0, "bad TMA box (%d,%d,%d) for C=%d", boxH, boxW, boxC, C);
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {(cuuint32_t)boxC, (cuuint32_t)boxW, (cuuint32_t)boxH, 1};
  return encode_bf16(map, 4, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}
int cvb_make_tmap_2d(CUtensorMap* map, const void* base, int64_t rows, int cols, int ld, int box_rows, int box_cols) {
  CVB_CHECK(box_rows > 0 && box_rows <= 256 && (box_cols == 32 || box_cols == 64) && ld % 8 == 0 && cols > 0 && rows > 0, "bad 2-D TMA box");
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  return encode_bf16(map, 2, base, dims, strides, box, box_cols == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B);
}

namespace {

constexpr int NT = 256;
// channels one CTA of a per-channel reduction covers (one 8-channel group per thread); wider maps add a grid dimension of channel chunks
constexpr int CH_CHUNK = 8 * NT;

// row-block geometry shared by the per-channel reduction kernels
struct RowGeom { int cgs, rpp, nthreads, rows_per_cta, ctas; };
RowGeom row_geom(int64_t M, int C) {
  RowGeom g;
  g.cgs = C / 8;
  g.rpp = NT / g.cgs; if (g.rpp < 1) g.rpp = 1;
  g.nthreads = g.cgs * g.rpp;
  int64_t target_ctas = 6 * (int64_t)cvb_num_sms();
  int64_t rows = (M + target_ctas - 1) / target_ctas;
  int64_t minrows = (int64_t)g.rpp * 4;
  if (rows < minrows) rows = minrows;
  rows = (rows + g.rpp - 1) / g.rpp * g.rpp;
  g.rows_per_cta = (int)rows;
  g.ctas = (int)((M + rows - 1) / rows);
  return g;
}

// ------------------------------------------------------------------------------------------------ tiny per-channel kernels
__global__ void bn_finalize_kernel(const double* sum, const double* sq, double count, const float* gamma, const float* beta, float eps,
                                   float momentum, float* rmean, float* rvar, int64_t* nbt, float* mean, float* rstd, float* scale,
                                   float* shift, int C) {
  pdl_wait();
  pdl_trigger();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0 && nbt) *nbt += 1;
  if (c >= C) return;
  double m = sum[c] / count;
  double var = sq[c] / count - m * m;
  if (var < 0) var = 0;
  float r = (float)(1.0 / sqrt(var + (double)eps));
  float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  mean[c] = (float)m;
  rstd[c] = r;
  scale[c] = g * r;
  shift[c] = b - (float)m * g * r;
  if (rmean) {
    double unbiased = count > 1 ? var * count / (count - 1) : var;
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)m;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unbiased;
  }
}

__global__ void bn_eval_kernel(const float* gamma, const float* beta, const float* rmean, const float* rvar, float eps, float* mean,
                               float* rstd, float* scale, float* shift, int C) {
  pdl_wait();
  pdl_trigger();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float r = rsqrtf(rvar[c] + eps);
  float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  mean[c] = rmean[c];
  rstd[c] = r;
  scale[c] = g * r;
  shift[c] = b - rmean[c] * g * r;
}

__global__ void bn_bwd_finalize_kernel(const double* sdz, const double* sdzy, double count, const float* gamma, const float* mean,
                                       const float* rstd, int eval_mode, float* dgamma, float* dbeta, float* c1, float* c2, float* c3,
                                       int C) {
  pdl_wait();
  pdl_trigger();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double db = sdz[c];
  double dg = (double)rstd[c] * (sdzy[c] - (double)mean[c] * sdz[c]);  // sum dz * xhat
  float g = gamma ? gamma[c] : 1.f;
  if (dgamma) dgamma[c] = (float)dg;
  if (dbeta) dbeta[c] = (float)db;
  float k1 = g * rstd[c];
  if (eval_mode) { c1[c] = k1; c2[c] = 0.f; c3[c] = 0.f; return; }
  // dy = g*rstd*(dz - db/n - xhat*dg/n),  xhat = (y-mean)*rstd
  double k2 = -(double)k1 * (double)rstd[c] * dg / count;
  double k3 = -(double)k1 * db / count - k2 * (double)mean[c];
  c1[c] = k1; c2[c] = (float)k2; c3[c] = (float)k3;
}

__global__ void gn_finalize_kernel(const double* ssum, const double* ssq, double count, float eps, float* mean, float* rstd, int B) {
  pdl_wait();
  pdl_trigger();
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double m = ssum[b] / count;
  double var = ssq[b] / count - m * m;
  if (var < 0) var = 0;
  mean[b] = (float)m;
  rstd[b] = (float)(1.0 / sqrt(var + (double)eps));
}

// ------------------------------------------------------------------------------------------------ elementwise: BN apply
__global__ void __launch_bounds__(NT) bn_apply_kernel(const bf16* __restrict__ Y, const float* __restrict__ scale, const float* __restrict__ shift,
                                                      int act, const bf16* __restrict__ R, bf16* __restrict__ OUT, int64_t nvec, int cgs) {
  pdl_wait();
  pdl_trigger();
  for (int64_t v = (int64_t)blockIdx.x * NT + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * NT) {
    int c = (int)(v % cgs) * 8;
    float f[8];
    unpack8(ldg16_stream(Y + v * 8), f);
    float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
    float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + c)), h1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
    float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    float sh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      f[j] = fmaf(sc[j], f[j], sh[j]);
      if (act) f[j] = silu_f(f[j]);
    }
    if (R) {
      float r[8];
      unpack8(ldg16_stream(R + v * 8), r);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] += r[j];
    }
    stg16(OUT + v * 8, pack8(f));
  }
}

// ------------------------------------------------------------------------------------------------ elementwise: operand load modes
// OUT[m, k] = load(A[, A2])[m, k]: materialises a prologue once for WIDE layers (many N tiles would each repeat it in the GEMM).
// Row-block geometry (row_geom): thread = (8-channel group, row lane); its per-channel parameters live in registers.
__global__ void __launch_bounds__(1024) apply_load_mode_rows_kernel(const bf16* __restrict__ A, const bf16* __restrict__ A2, int mode,
                                                                    const float* __restrict__ p0, const float* __restrict__ p1,
                                                                    const float* __restrict__ p2, const float* __restrict__ row_mean,
                                                                    const float* __restrict__ row_rstd, int rps, bf16* __restrict__ OUT, int M, int cgs,
                                                                    int rpp, int rows_per_cta, int lda, int lda2, int ldo) {
  pdl_wait();
  pdl_trigger();
  const int cg = threadIdx.x % cgs, rr = threadIdx.x / cgs;
  const int c = cg * 8;
  float q0[8], q1[8], q2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    q0[j] = p0 ? __ldg(p0 + c + j) : 1.f;
    q1[j] = p1 ? __ldg(p1 + c + j) : 0.f;
    q2[j] = (mode == CVB_A_BNB && p2) ? __ldg(p2 + c + j) : 0.f;
  }
  const int r_begin = blockIdx.x * rows_per_cta;
  const int r_end = min(M, r_begin + rows_per_cta);
#pragma unroll 4
  for (int r = r_begin + rr; r < r_end; r += rpp) {
    float f[8];
    unpack8(ldg16_stream(A + (size_t)r * lda + c), f);
    if (mode == CVB_A_BNB) {
      float y[8];
      unpack8(ldg16_stream(A2 + (size_t)r * lda2 + c), y);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaf(q0[j], f[j], fmaf(q1[j], y[j], q2[j]));
    } else if (mode == CVB_A_GN) {
      const int b = r / rps;
      const float mu = __ldg(row_mean + b), rs = __ldg(row_rstd + b);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaf((f[j] - mu) * rs, q0[j], q1[j]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = apply_mode(mode, f[j], q0[j], q1[j]);
    }
    stg16(OUT + (size_t)r * ldo + c, pack8(f));
  }
}

// ------------------------------------------------------------------------------------------------ per-channel reductions
// mode 0: BN backward reduce: dz = dout (act 0) or dout*silu'(sc*y+sh) (act 1); s0 += dz, s1 += dz*y; optional DZ store.
__global__ void __launch_bounds__(NT) bn_bwd_reduce_kernel(const bf16* __restrict__ DOUT, const bf16* __restrict__ Y, const float* __restrict__ scale,
                                                           const float* __restrict__ shift, int act, bf16* __restrict__ DZ, double* s0, double* s1,
                                                           int64_t M, int C, int rows_per_cta) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ double sdred[];  // fp64: the threads' fp32 partials add exactly, whatever the order; [2][nc]
  const int tid = threadIdx.x;
  // grid: (row blocks, channel chunks); thread = (8-channel group of the chunk, row lane)
  const int c0 = blockIdx.y * CH_CHUNK, nc = min(C - c0, CH_CHUNK), cgs = nc / 8, rpp = blockDim.x / cgs;
  for (int i = tid; i < 2 * nc; i += blockDim.x) sdred[i] = 0.0;
  __syncthreads();
  const int cg = tid % cgs, rr = tid / cgs;
  const int c = c0 + cg * 8;
  float sc[8], sh[8], a0[8], a1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { sc[j] = act ? scale[c + j] : 1.f; sh[j] = act ? shift[c + j] : 0.f; a0[j] = 0.f; a1[j] = 0.f; }
  int64_t r_begin = (int64_t)blockIdx.x * rows_per_cta, r_end = r_begin + rows_per_cta;
  if (r_end > M) r_end = M;
  if (rr >= rpp) r_end = r_begin;  // the threads past cgs * rpp of a narrower last chunk
  for (int64_t r = r_begin + rr; r < r_end; r += rpp) {
    float d[8], y[8];
    unpack8(ldg16_stream(DOUT + r * C + c), d);
    unpack8(ldg16_stream(Y + r * C + c), y);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (act) d[j] = bf16_round(d[j] * silu_grad_f(fmaf(sc[j], y[j], sh[j])));
      a0[j] += d[j];
      a1[j] += d[j] * y[j];
    }
    if (DZ) stg16(DZ + r * C + c, pack8(d));
  }
  if (rr < rpp) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { atomicAdd(&sdred[cg * 8 + j], (double)a0[j]); atomicAdd(&sdred[nc + cg * 8 + j], (double)a1[j]); }
  }
  __syncthreads();
  for (int i = tid; i < nc; i += blockDim.x) { atomicAdd(s0 + c0 + i, sdred[i]); atomicAdd(s1 + c0 + i, sdred[nc + i]); }
}

// per-sample sum / sumsq
__global__ void __launch_bounds__(NT) gn_stats_kernel(const bf16* __restrict__ X, int ldx, int rows_per_sample, int C, int chunks_per_sample,
                                                      double* ssum, double* ssq) {
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.x / chunks_per_sample, chunk = blockIdx.x % chunks_per_sample;
  const int cgs = C / 8;
  const int64_t nvec = (int64_t)rows_per_sample * cgs;
  const int64_t per = (nvec + chunks_per_sample - 1) / chunks_per_sample;
  int64_t v0 = chunk * per, v1 = v0 + per;
  if (v1 > nvec) v1 = nvec;
  float s = 0.f, q = 0.f;
  for (int64_t v = v0 + threadIdx.x; v < v1; v += NT) {
    int64_t r = v / cgs;
    int c = (int)(v % cgs) * 8;
    float f[8];
    unpack8(ldg16_stream(X + ((int64_t)b * rows_per_sample + r) * ldx + c), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { s += f[j]; q += f[j] * f[j]; }
  }
  __shared__ float ws[2][NT / 32];
  s = warp_sum(s); q = warp_sum(q);
  if ((threadIdx.x & 31) == 0) { ws[0][threadIdx.x >> 5] = s; ws[1][threadIdx.x >> 5] = q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ts = 0.f, tq = 0.f;
    for (int i = 0; i < NT / 32; ++i) { ts += ws[0][i]; tq += ws[1][i]; }
    atomicAdd(ssum + b, (double)ts);
    atomicAdd(ssq + b, (double)tq);
  }
}

// Stand-alone GroupNorm(1, C) backward, phase 1 (when no producing GEMM epilogue took the sums): per-channel dbeta += v, dgamma += v*xhat and
// per-sample sums of g = v*gamma and g*xhat.  CTA = (row chunk, sample); a thread owns one 8-channel group.
__global__ void __launch_bounds__(NT) gn_bwd_stats_kernel(const bf16* __restrict__ V, const bf16* __restrict__ X, const float* __restrict__ mean,
                                                          const float* __restrict__ rstd, const float* __restrict__ gamma, int rows_per_sample, int C,
                                                          int cgs, int rpp, int rows_per_cta, double* dgamma, double* dbeta, double* sg, double* sgx) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ double sdred[];  // fp64: the threads' fp32 partials add exactly, whatever the order; [2][C]
  __shared__ float ws[2][NT / 32];
  const int tid = threadIdx.x, b = blockIdx.y;
  for (int i = tid; i < 2 * C; i += blockDim.x) sdred[i] = 0.0;
  __syncthreads();
  const int cg = tid % cgs, rr = tid / cgs, c = cg * 8;
  const float mu = mean[b], rs = rstd[b];
  float db[8], dg[8], gm[8], s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) { db[j] = 0.f; dg[j] = 0.f; gm[j] = gamma[c + j]; }
  int r_begin = blockIdx.x * rows_per_cta, r_end = r_begin + rows_per_cta;
  if (r_end > rows_per_sample) r_end = rows_per_sample;
  if (rr < rpp) {
    for (int r = r_begin + rr; r < r_end; r += rpp) {
      const int64_t row = (int64_t)b * rows_per_sample + r;
      float v[8], x[8];
      unpack8(ldg16_stream(V + row * C + c), v);
      unpack8(ldg16_stream(X + row * C + c), x);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (x[j] - mu) * rs, g = v[j] * gm[j];
        db[j] += v[j];
        dg[j] = fmaf(v[j], xh, dg[j]);
        s1 += g;
        s2 = fmaf(g, xh, s2);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { atomicAdd(&sdred[c + j], (double)db[j]); atomicAdd(&sdred[C + c + j], (double)dg[j]); }
  }
  s1 = warp_sum(s1); s2 = warp_sum(s2);
  if ((tid & 31) == 0) { ws[0][tid >> 5] = s1; ws[1][tid >> 5] = s2; }
  __syncthreads();
  for (int i = tid; i < C; i += blockDim.x) { atomicAdd(dbeta + i, sdred[i]); atomicAdd(dgamma + i, sdred[C + i]); }
  if (tid == 0) {
    float a = 0.f, q = 0.f;
    for (int i = 0; i < (int)(blockDim.x + 31) / 32; ++i) { a += ws[0][i]; q += ws[1][i]; }
    atomicAdd(sg + b, (double)a);
    atomicAdd(sgx + b, (double)q);
  }
}

// GroupNorm backward phase 2 (+ residual-stream gradient, + column sums of the result)
// LayerNorm backward in ONE pass (a "sample" is a single token row, so both phases of the GroupNorm backward fit in a warp):
//   g = v * gamma;  dx = rstd * (g - mean_c(g) - xhat * mean_c(g * xhat)) + dres;   dbeta += v;  dgamma += v * xhat;  col_sum += dx
// (autograd of nn.LayerNorm, cvnets/layers/normalization/layer_norm.py:14-72).  One warp per row, rows grid-strided; the per-channel
// sums live in shared memory and are flushed once per CTA.  A row stays in registers: lane owns 8-channel chunks lane, lane+32, ..., MAXCH of
// them, so C <= 256 * MAXCH.  MAXCH = 4 serves C <= 1024; MAXCH = 5 the 1280-wide ViT-H rows (the widest LayerNorm of any recipe).
constexpr int LNB_MAXCH = 5;
template <int MAXCH>
__global__ void __launch_bounds__(NT) ln_bwd_kernel(const bf16* __restrict__ V, const bf16* __restrict__ X, const float* __restrict__ mean,
                                                    const float* __restrict__ rstd, const float* __restrict__ gamma, const bf16* __restrict__ DRES,
                                                    bf16* __restrict__ DX, int64_t M, int C, double* dgamma, double* dbeta, double* col_sum) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sred[];  // [3][C] per-channel sums of the CTA (dbeta, dgamma, column sums of DX) + [C] gamma
  float* sgam = sred + 3 * C;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 3 * C; i += NT) sred[i] = 0.f;
  for (int i = tid; i < C; i += NT) sgam[i] = gamma[i];
  __syncthreads();
  const int nch = C / 8;
  // The per-channel sums go to shared memory with one reduction per (row, channel): keeping them in registers (96 accumulators per lane at C = 768)
  // cost 246 registers = 8 warps per SM
  const float invC = 1.0f / (float)C;
  for (int64_t row = (int64_t)blockIdx.x * (NT / 32) + warp; row < M; row += (int64_t)gridDim.x * (NT / 32)) {
    const float mu = mean[row], rs = rstd[row];
    float v[MAXCH][8], xh[MAXCH][8];
    uint4 dres[MAXCH];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int q = 0; q < MAXCH; ++q) {
      const int ch = lane + 32 * q;
      if (ch < nch) {
        unpack8(ldg16_stream(V + row * C + ch * 8), v[q]);
        unpack8(ldg16_stream(X + row * C + ch * 8), xh[q]);
        if (DRES) dres[q] = ldg16_stream(DRES + row * C + ch * 8);  // issued with the other loads, consumed after the row reduction
      }
    }
#pragma unroll
    for (int q = 0; q < MAXCH; ++q) {
      const int ch = lane + 32 * q;
      if (ch < nch) {
        float gq[8];
        *reinterpret_cast<float4*>(gq) = *reinterpret_cast<const float4*>(sgam + ch * 8);
        *reinterpret_cast<float4*>(gq + 4) = *reinterpret_cast<const float4*>(sgam + ch * 8 + 4);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          xh[q][e] = (xh[q][e] - mu) * rs;
          atomicAdd(&sred[e * nch + ch], v[q][e]);  // [element][chunk] layout: the 32 lanes of a reduction hit 32 different banks
          atomicAdd(&sred[C + e * nch + ch], v[q][e] * xh[q][e]);
          v[q][e] *= gq[e];  // from here on v holds g = V * gamma
          s1 += v[q][e];
          s2 = fmaf(v[q][e], xh[q][e], s2);
        }
      }
    }
    s1 = warp_sum(s1) * invC;
    s2 = warp_sum(s2) * invC;
#pragma unroll
    for (int q = 0; q < MAXCH; ++q) {
      const int ch = lane + 32 * q;
      if (ch < nch) {
        float d[8];
        if (DRES) unpack8(dres[q], d);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float o = rs * (v[q][e] - s1 - xh[q][e] * s2);
          if (DRES) o += d[e];
          d[e] = o;
          if (col_sum) atomicAdd(&sred[2 * C + e * nch + ch], o);
        }
        stg16(DX + row * C + ch * 8, pack8(d));
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < C; i += NT) {
    const int t = (i & 7) * (C / 8) + (i >> 3);  // channel i lives at [element i % 8][chunk i / 8]
    atomicAdd(dbeta + i, (double)sred[t]);
    atomicAdd(dgamma + i, (double)sred[C + t]);
    if (col_sum) atomicAdd(col_sum + i, (double)sred[2 * C + t]);
  }
}

// stand-alone activation passes for the transformer FFN when the activation is not SiLU (GELU of the ViT / CLIP recipes; the
// SiLU FFN keeps the activation fused into the GEMM load / epilogue modes; Hardswish / Hardsigmoid: the MobileNetv3-style InvertedResidualSE
// block, cvnets/modules/mobilenetv2.py:16-138).  kind: CVB_ACT_*; the default branch is CVB_ACT_SIGMOID.
__device__ __forceinline__ float act_fwd_f(float x, int kind) {
  switch (kind) {
    case CVB_ACT_SILU: return silu_f(x);
    case CVB_ACT_GELU: return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
    case CVB_ACT_RELU: return fmaxf(x, 0.f);
    case CVB_ACT_HARDSWISH: return x * fminf(fmaxf(x + 3.0f, 0.f), 6.0f) * (1.0f / 6.0f);
    case CVB_ACT_HARDSIGMOID: return fminf(fmaxf(x + 3.0f, 0.f), 6.0f) * (1.0f / 6.0f);
    default: return 1.0f / (1.0f + __expf(-x));
  }
}
__device__ __forceinline__ float act_grad_f(float x, int kind) {
  switch (kind) {
    case CVB_ACT_SILU: return silu_grad_f(x);
    case CVB_ACT_GELU: {
      const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
      return cdf + x * 0.3989422804014327f * __expf(-0.5f * x * x);
    }
    case CVB_ACT_RELU: return x > 0.f ? 1.f : 0.f;
    case CVB_ACT_HARDSWISH: return x <= -3.0f ? 0.f : (x < 3.0f ? fmaf(x, 1.0f / 3.0f, 0.5f) : 1.0f);  // torch's hardswish_backward: 0 at -3, 1 at 3
    case CVB_ACT_HARDSIGMOID: return (x > -3.0f && x < 3.0f) ? (1.0f / 6.0f) : 0.f;
    default: {
      const float s = 1.0f / (1.0f + __expf(-x));
      return s * (1.0f - s);
    }
  }
}
__global__ void __launch_bounds__(NT) act_fwd_kernel(const bf16* __restrict__ X, bf16* __restrict__ Y, int64_t nvec, int kind) {
  pdl_wait();
  pdl_trigger();
  for (int64_t v = (int64_t)blockIdx.x * NT + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * NT) {
    float f[8];
    unpack8(ldg16_stream(X + v * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = act_fwd_f(f[j], kind);
    stg16(Y + v * 8, pack8(f));
  }
}
__global__ void __launch_bounds__(NT) act_bwd_kernel(const bf16* __restrict__ DY, const bf16* __restrict__ X, bf16* __restrict__ DX, int64_t nvec,
                                                     int kind) {
  pdl_wait();
  pdl_trigger();
  for (int64_t v = (int64_t)blockIdx.x * NT + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * NT) {
    float g[8], x[8];
    unpack8(ldg16_stream(DY + v * 8), g);
    unpack8(ldg16_stream(X + v * 8), x);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= act_grad_f(x[j], kind);
    stg16(DX + v * 8, pack8(g));
  }
}

// LayerNorm statistics: one warp per token row
__global__ void __launch_bounds__(NT) ln_stats_kernel(const bf16* __restrict__ X, int ldx, int64_t M, int C, float eps, float* __restrict__ mean,
                                                      float* __restrict__ rstd) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (NT / 32) + (threadIdx.x >> 5);
  if (row >= M) return;
  const bf16* x = X + row * ldx;
  float s = 0.f, q = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    float f[8];
    unpack8(ldg16(x + c), f);
#pragma unroll
    for (int e = 0; e < 8; ++e) { s += f[e]; q = fmaf(f[e], f[e], q); }
  }
  s = warp_sum(s);
  q = warp_sum(q);
  if (lane == 0) {
    const float mu = s / (float)C;
    float var = q / (float)C - mu * mu;
    if (var < 0.f) var = 0.f;
    mean[row] = mu;
    rstd[row] = rsqrtf(var + eps);
  }
}

// Row-block geometry (row_geom): thread = (8-channel group cg, row lane rr) walks rows r_begin + rr, + rpp, ... of its CTA's run.  That walk
// fixes the fp32 chain of each column partial; the loads of GNB_U consecutive steps are issued before any of them is used, so a thread has
// up to 3 * GNB_U 16-byte loads in flight.  b is constant over most of a run of rows: the per-sample terms are recomputed only where a thread's
// rows cross into the next sample.
constexpr int GNB_U = 2;
__global__ void __launch_bounds__(NT) gn_bwd_apply_kernel(const bf16* __restrict__ G, const bf16* __restrict__ X, const float* __restrict__ mean,
                                                          const float* __restrict__ rstd, const double* __restrict__ sg, const double* __restrict__ sgx,
                                                          double count, const bf16* __restrict__ DRES, bf16* __restrict__ DX, int64_t M,
                                                          int rows_per_sample, int C, double* col_sum, int cgs, int rpp, int rows_per_cta,
                                                          const float* __restrict__ gamma) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float spart[];  // [rpp][C]: the threads' fp32 column partials, added in fp64 in a fixed order
  const int tid = threadIdx.x;
  const int cg = tid % cgs, rr = tid / cgs;
  const int c = cg * 8;
  float a0[8], gm[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { a0[j] = 0.f; gm[j] = gamma ? gamma[c + j] : 1.0f; }
  const int64_t r_begin = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t r_end = r_begin + rows_per_cta < M ? r_begin + rows_per_cta : M;
  int64_t r = r_begin + rr;
  int b = (int)(r / rows_per_sample);
  int64_t b_end = (int64_t)(b + 1) * rows_per_sample;  // first row of sample b + 1
  float mu = 0.f, rs = 0.f, m1 = 0.f, m2 = 0.f;
  if (r < r_end) { mu = mean[b]; rs = rstd[b]; m1 = (float)(sg[b] / count); m2 = (float)(sgx[b] / count); }
  for (; r < r_end; r += GNB_U * rpp) {
    uint4 gv[GNB_U], xv[GNB_U], dv[GNB_U];
#pragma unroll
    for (int u = 0; u < GNB_U; ++u) {
      const int64_t ru = r + (int64_t)u * rpp;
      if (ru < r_end) {
        gv[u] = ldg16_stream(G + ru * C + c);
        xv[u] = ldg16_stream(X + ru * C + c);
        if (DRES) dv[u] = ldg16_stream(DRES + ru * C + c);
      }
    }
#pragma unroll
    for (int u = 0; u < GNB_U; ++u) {
      const int64_t ru = r + (int64_t)u * rpp;
      if (ru >= r_end) break;
      if (ru >= b_end) {
        do { ++b; b_end += rows_per_sample; } while (ru >= b_end);
        mu = mean[b]; rs = rstd[b]; m1 = (float)(sg[b] / count); m2 = (float)(sgx[b] / count);
      }
      float g[8], x[8];
      unpack8(gv[u], g);
      unpack8(xv[u], x);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float xh = (x[j] - mu) * rs;
        g[j] = rs * (g[j] * gm[j] - m1 - xh * m2);
      }
      if (DRES) {
        float d[8];
        unpack8(dv[u], d);
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] += d[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) a0[j] += g[j];  // column sums (bias gradients) from the unrounded fp32 values
      stg16(DX + ru * C + c, pack8(g));
    }
  }
  if (col_sum) {
    float4* dst = reinterpret_cast<float4*>(spart + rr * C + c);
    dst[0] = make_float4(a0[0], a0[1], a0[2], a0[3]);
    dst[1] = make_float4(a0[4], a0[5], a0[6], a0[7]);
    __syncthreads();
    for (int i = tid; i < C; i += blockDim.x) {
      double t = 0.0;
      for (int q = 0; q < rpp; ++q) t += (double)spart[q * C + i];
      atomicAdd(col_sum + i, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------ global average pool
__global__ void __launch_bounds__(NT) pool_fwd_kernel(const bf16* __restrict__ X, int HW, int C, bf16* __restrict__ OUT) {
  pdl_wait();
  pdl_trigger();
  // grid: (B, channel chunks); thread = (8-channel group of the chunk, row lane)
  extern __shared__ double sdred[];  // fp64: the threads' fp32 partials add exactly, whatever the order; [nc]
  const int b = blockIdx.x;
  const int c0 = blockIdx.y * CH_CHUNK, nc = min(C - c0, CH_CHUNK), cgs = nc / 8;
  const int tid = threadIdx.x;
  for (int i = tid; i < nc; i += blockDim.x) sdred[i] = 0.0;
  __syncthreads();
  const int cg = tid % cgs, rr = tid / cgs, rpp = blockDim.x / cgs;
  if (rr < rpp) {  // the threads past cgs * rpp of a narrower last chunk have no rows
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = 0.f;
    for (int r = rr; r < HW; r += rpp) {
      float f[8];
      unpack8(ldg16(X + ((int64_t)b * HW + r) * C + c0 + cg * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += f[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) atomicAdd(&sdred[cg * 8 + j], (double)a[j]);
  }
  __syncthreads();
  for (int i = tid; i < nc; i += blockDim.x) OUT[(int64_t)b * C + c0 + i] = __float2bfloat16_rn((float)sdred[i] / (float)HW);
}

__global__ void __launch_bounds__(NT) pool_bwd_kernel(const bf16* __restrict__ DOUT, int HW, int C, bf16* __restrict__ DX, int64_t nvec) {
  pdl_wait();
  pdl_trigger();
  const int cgs = C / 8;
  const float inv = 1.f / (float)HW;
  for (int64_t v = (int64_t)blockIdx.x * NT + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * NT) {
    int64_t row = v / cgs;
    int c = (int)(v % cgs) * 8;
    int64_t b = row / HW;
    float f[8];
    unpack8(ldg16(DOUT + b * C + c), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= inv;
    stg16(DX + v * 8, pack8(f));
  }
}

// ------------------------------------------------------------------------------------------------ stem im2col
// A[(b,oh,ow), ci*9+u*3+v] = bf16(X[b,ci,2oh+u-1,2ow+v-1]) (zero padded), columns 27..31 = 0
// mix (device, 6 floats, may be NULL): {mode, lambda, x1, y1, x2, y2} -- the batch-mixing transforms of the reference's input edge
// (data/transforms/image_torch.py:99-137 RandomMixup, :290-342 RandomCutmix; applied at engine/training_engine.py:236-238) folded into the
// gather: every sample is paired with its predecessor in the batch (image.roll(1, 0)); mode 1: x = lambda*x + (1-lambda)*x_prev (fp32, as the
// reference), mode 2: the box [y1,y2) x [x1,x2) is pasted from x_prev.  No extra pass over the images, no mixed copy in HBM.
__global__ void __launch_bounds__(NT) stem_im2col_kernel(const float* __restrict__ X, int64_t sxn, int64_t sxc, int64_t sxh, int64_t sxw, int B, int H,
                                                         int W, bf16* __restrict__ A, const float* __restrict__ mix) {
  pdl_wait();
  pdl_trigger();
  const int Ho = H / 2, Wo = W / 2;
  const int mode = mix ? (int)mix[0] : 0;
  const float lam = mix ? mix[1] : 1.f;
  const int bx1 = mix ? (int)mix[2] : 0, by1 = mix ? (int)mix[3] : 0, bx2 = mix ? (int)mix[4] : 0, by2 = mix ? (int)mix[5] : 0;
  const int64_t total = (int64_t)B * Ho * Wo * 4;  // 4 chunks of 8 columns per output pixel
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    const int ch = (int)(i & 3);
    const int64_t pix = i >> 2;
    const int ow = (int)(pix % Wo);
    const int oh = (int)((pix / Wo) % Ho);
    const int b = (int)(pix / ((int64_t)Wo * Ho));
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = ch * 8 + j;
      float v = 0.f;
      if (col < 27) {
        const int ci = col / 9, u = (col % 9) / 3, vv = col % 3;
        const int h = 2 * oh + u - 1, w = 2 * ow + vv - 1;
        if (h >= 0 && h < H && w >= 0 && w < W) {
          const int64_t off = ci * sxc + h * sxh + w * sxw;
          v = __ldg(X + b * sxn + off);
          if (mode != 0) {
            const int bp = b == 0 ? B - 1 : b - 1;
            if (mode == 1) v = fmaf(lam, v, (1.0f - lam) * __ldg(X + bp * sxn + off));
            else if (h >= by1 && h < by2 && w >= bx1 && w < bx2) v = __ldg(X + bp * sxn + off);
          }
        }
      }
      f[j] = v;
    }
    stg16(A + i * 8, pack8(f));
  }
}

// ------------------------------------------------------------------------------------------------ weight preparation
__device__ __forceinline__ int perm_row(int r, int rows, int rot) { return rot ? (r + rot) % rows : r; }

__global__ void __launch_bounds__(NT) prep_weights_kernel(const cvb_prep_desc* __restrict__ descs) {
  pdl_wait();
  pdl_trigger();
  const cvb_prep_desc d = descs[blockIdx.y];
  const int64_t total = (d.kind == CVB_PREP_TAPMAJOR_F32) ? (int64_t)d.rows * d.cols
                        : (d.kind == CVB_PREP_VECTOR_F32 ? (int64_t)d.dst_rows : (int64_t)d.dst_rows * d.ldd);
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    if (d.kind == CVB_PREP_ROWMAJOR) {
      int r = (int)(i / d.ldd), c = (int)(i % d.ldd);
      float v = (r < d.rows && c < d.cols) ? d.src[(int64_t)perm_row(r, d.rows, d.rot) * d.cols + c] : 0.f;
      static_cast<bf16*>(d.dst)[i] = __float2bfloat16_rn(v);
    } else if (d.kind == CVB_PREP_TRANSPOSED) {
      int c = (int)(i / d.ldd), r = (int)(i % d.ldd);
      float v = (r < d.rows && c < d.cols) ? d.src[(int64_t)perm_row(r, d.rows, d.rot) * d.cols + c] : 0.f;
      static_cast<bf16*>(d.dst)[i] = __float2bfloat16_rn(v);
    } else if (d.kind == CVB_PREP_TAPMAJOR_F32) {
      int tap = (int)(i / d.rows), ch = (int)(i % d.rows);
      static_cast<float*>(d.dst)[i] = bf16_round(d.src[(int64_t)ch * d.cols + tap]);
    } else if (d.kind == CVB_PREP_PATCH || d.kind == CVB_PREP_PATCH_T) {
      // dense conv weight [rows = Cout][cols = Cin * taps] in (ci, tap) order -> patch-matrix order (tap, ci); rot = taps.
      // PATCH: row-major [dst_rows, ldd];  PATCH_T: transposed [cols, ldd >= rows]
      const int r = (d.kind == CVB_PREP_PATCH) ? (int)(i / d.ldd) : (int)(i % d.ldd), c = (d.kind == CVB_PREP_PATCH) ? (int)(i % d.ldd) : (int)(i / d.ldd);
      const int cin = d.cols / d.rot;
      float v = 0.f;
      if (r < d.rows && c < d.cols) v = d.src[(int64_t)r * d.cols + (c % cin) * d.rot + c / cin];
      static_cast<bf16*>(d.dst)[i] = __float2bfloat16_rn(v);
    } else {  // CVB_PREP_VECTOR_F32
      int r = (int)i;
      static_cast<float*>(d.dst)[i] = (r < d.rows) ? d.src[perm_row(r, d.rows, d.rot)] : 0.f;
    }
  }
}

__global__ void __launch_bounds__(NT) unprep_grad_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols, int lds, int kind,
                                                         int rot) {
  pdl_wait();
  pdl_trigger();
  const int64_t total = (int64_t)rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    if (kind == CVB_PREP_ROWMAJOR) {
      int r = (int)(i / cols), c = (int)(i % cols);
      dst[(int64_t)perm_row(r, rows, rot) * cols + c] = src[(int64_t)r * lds + c];
    } else if (kind == CVB_PREP_TAPMAJOR_F32) {  // src [taps=cols][C=rows] -> dst [C][taps]
      int ch = (int)(i / cols), tap = (int)(i % cols);
      dst[i] = src[(int64_t)tap * rows + ch];
    } else if (kind == CVB_PREP_PATCH) {  // src [rows][(tap, ci)] (leading dim lds) -> dst [rows][(ci, tap)], rot = taps
      int r = (int)(i / cols), c = (int)(i % cols);
      const int cin = cols / rot;
      dst[(int64_t)r * cols + (c % cin) * rot + c / cin] = src[(int64_t)r * lds + c];
    } else {  // CVB_PREP_VECTOR_F32
      dst[perm_row((int)i, rows, rot)] = src[i];
    }
  }
}

int grid_for(int64_t n_items) {
  int64_t g = (n_items + NT - 1) / NT;
  int64_t cap = 16 * (int64_t)cvb_num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

extern "C" int cvb_bn_finalize(const double* sum, const double* sq, double count, const float* gamma, const float* beta, float eps, float momentum,
                               float* running_mean, float* running_var, int64_t* nbt, float* mean, float* rstd, float* scale, float* shift, int C,
                               cvb_stream_t stream) {
  CVB_CHECK(sum && sq && mean && rstd && scale && shift && C > 0 && count > 0, "cvb_bn_finalize: bad arguments");
  CVB_CUDA(cvb_launch(bn_finalize_kernel, (C + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream), sum, sq, count, gamma, beta, eps, momentum, running_mean,
                                                                                     running_var, nbt, mean, rstd, scale, shift, C));
  return 0;
}

extern "C" int cvb_bn_eval_scale_shift(const float* gamma, const float* beta, const float* running_mean, const float* running_var, float eps,
                                       float* mean, float* rstd, float* scale, float* shift, int C, cvb_stream_t stream) {
  CVB_CHECK(running_mean && running_var && mean && rstd && scale && shift && C > 0, "cvb_bn_eval_scale_shift: bad arguments");
  CVB_CUDA(cvb_launch(bn_eval_kernel, (C + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream), gamma, beta, running_mean, running_var, eps, mean, rstd, scale, shift, C));
  return 0;
}

extern "C" int cvb_bn_bwd_finalize(const double* sum_dz, const double* sum_dzy, double count, const float* gamma, const float* mean, const float* rstd,
                                   int eval_mode, float* dgamma, float* dbeta, float* c1, float* c2, float* c3, int C, cvb_stream_t stream) {
  CVB_CHECK(sum_dz && sum_dzy && mean && rstd && c1 && c2 && c3 && C > 0 && count > 0, "cvb_bn_bwd_finalize: bad arguments");
  CVB_CUDA(cvb_launch(bn_bwd_finalize_kernel, (C + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream), sum_dz, sum_dzy, count, gamma, mean, rstd, eval_mode, dgamma,
                                                                                         dbeta, c1, c2, c3, C));
  return 0;
}

extern "C" int cvb_bn_apply(const void* Y, const float* scale, const float* shift, int act, const void* R, void* OUT, int64_t M, int C,
                            cvb_stream_t stream) {
  CVB_CHECK(Y && scale && shift && OUT && M > 0 && C > 0 && C % 8 == 0, "cvb_bn_apply: bad arguments");
  int64_t nvec = M * (C / 8);
  CVB_CUDA(cvb_launch(bn_apply_kernel, grid_for(nvec), NT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(Y), scale, shift, act,
                                                                               static_cast<const bf16*>(R), static_cast<bf16*>(OUT), nvec, C / 8));
  return 0;
}

extern "C" int cvb_apply_load_mode(const void* A, int lda, const void* A2, int lda2, int mode, const float* p0, const float* p1, const float* p2,
                                   const float* row_mean, const float* row_rstd, int rows_per_sample, void* OUT, int ldo, int64_t M, int K,
                                   cvb_stream_t stream) {
  CVB_CHECK(A && OUT && M > 0 && K > 0 && K % 8 == 0 && lda % 8 == 0 && ldo % 8 == 0, "cvb_apply_load_mode: bad arguments");
  CVB_CHECK(K <= 8192 && M < (int64_t)1 << 31, "cvb_apply_load_mode: K = %d, M = %lld (at most 8192 channels and 2^31 - 1 rows)", K, (long long)M);
  CVB_CHECK(mode >= CVB_A_AFF && mode <= CVB_A_BNB, "cvb_apply_load_mode: mode %d", mode);
  if (mode == CVB_A_BNB) CVB_CHECK(A2 && p0 && p1 && p2 && lda2 % 8 == 0, "cvb_apply_load_mode: BNB needs A2 and p0/p1/p2");
  if (mode == CVB_A_GN) CVB_CHECK(row_mean && row_rstd && rows_per_sample > 0 && p0 && p1, "cvb_apply_load_mode: GN needs statistics");
  if (mode == CVB_A_AFF || mode == CVB_A_AFF_SILU) CVB_CHECK(p0 && p1, "cvb_apply_load_mode: AFF needs p0/p1");
  RowGeom g = row_geom(M, K);
  CVB_CUDA(cvb_launch(apply_load_mode_rows_kernel, g.ctas, g.nthreads, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(A),
                      static_cast<const bf16*>(A2), mode, p0, p1, p2, row_mean, row_rstd, rows_per_sample > 0 ? rows_per_sample : 1,
                      static_cast<bf16*>(OUT), (int)M, g.cgs, g.rpp, g.rows_per_cta, lda, lda2, ldo));
  return 0;
}

extern "C" int cvb_bn_bwd_reduce(const void* DOUT, const void* Y, const float* scale, const float* shift, int act, void* DZ, double* sum_dz,
                                 double* sum_dzy, int64_t M, int C, cvb_stream_t stream) {
  CVB_CHECK(DOUT && Y && sum_dz && sum_dzy && M > 0 && C > 0 && C % 8 == 0, "cvb_bn_bwd_reduce: bad arguments");
  if (act) CVB_CHECK(scale && shift, "cvb_bn_bwd_reduce: act needs scale/shift");
  const int nc = C < CH_CHUNK ? C : CH_CHUNK;
  RowGeom g = row_geom(M, nc);
  CVB_CUDA(cvb_launch(bn_bwd_reduce_kernel, dim3(g.ctas, (C + CH_CHUNK - 1) / CH_CHUNK), g.nthreads, 2 * nc * sizeof(double),
      static_cast<cudaStream_t>(stream), static_cast<const bf16*>(DOUT), static_cast<const bf16*>(Y), scale, shift, act, static_cast<bf16*>(DZ), sum_dz,
      sum_dzy, M, C, g.rows_per_cta));
  return 0;
}

extern "C" int cvb_gn_finalize(const double* samp_sum, const double* samp_sq, double count, float eps, float* mean, float* rstd, int B,
                               cvb_stream_t stream) {
  CVB_CHECK(samp_sum && samp_sq && mean && rstd && B > 0 && count > 0, "cvb_gn_finalize: bad arguments");
  CVB_CUDA(cvb_launch(gn_finalize_kernel, (B + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream), samp_sum, samp_sq, count, eps, mean, rstd, B));
  return 0;
}

extern "C" int cvb_gn_stats(const void* X, int ldx, int B, int rows_per_sample, int C, double* samp_sum, double* samp_sq, cvb_stream_t stream) {
  CVB_CHECK(X && samp_sum && samp_sq && B > 0 && rows_per_sample > 0 && C > 0 && C % 8 == 0 && ldx % 8 == 0, "cvb_gn_stats: bad arguments");
  int64_t nvec = (int64_t)rows_per_sample * (C / 8);
  int chunks = (int)((nvec + 4095) / 4096);
  if (chunks < 1) chunks = 1;
  CVB_CUDA(cvb_launch(gn_stats_kernel, B * chunks, NT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(X), ldx, rows_per_sample, C, chunks, samp_sum,
                                                                           samp_sq));
  return 0;
}

extern "C" int cvb_ln_bwd(const void* V, const void* X, const float* mean, const float* rstd, const float* gamma, const void* DRES, void* DX,
                          int64_t M, int C, double* dgamma, double* dbeta, double* col_sum, cvb_stream_t stream) {
  CVB_CHECK(V && X && mean && rstd && gamma && DX && dgamma && dbeta && M > 0 && C > 0 && C % 8 == 0, "cvb_ln_bwd: bad arguments");
  CVB_CHECK(C <= 256 * LNB_MAXCH, "cvb_ln_bwd: C = %d > %d is not supported", C, 256 * LNB_MAXCH);
  CVB_CHECK(cvb_aligned16(V) && cvb_aligned16(X) && cvb_aligned16(DX) && (!DRES || cvb_aligned16(DRES)), "cvb_ln_bwd: misaligned operand");
  int64_t ctas = (M + NT / 32 - 1) / (NT / 32);
  const int64_t cap = 4 * (int64_t)cvb_num_sms();
  if (ctas > cap) ctas = cap;
  CVB_CUDA(cvb_launch(C <= 1024 ? ln_bwd_kernel<4> : ln_bwd_kernel<LNB_MAXCH>, (unsigned)ctas, NT, (size_t)4 * C * sizeof(float), static_cast<cudaStream_t>(stream), static_cast<const bf16*>(V),
                      static_cast<const bf16*>(X), mean, rstd, gamma, static_cast<const bf16*>(DRES), static_cast<bf16*>(DX), M, C, dgamma, dbeta,
                      col_sum));
  return 0;
}

extern "C" int cvb_act_fwd(const void* X, void* Y, int64_t n, int kind, cvb_stream_t stream) {
  CVB_CHECK(X && Y && n > 0 && n % 8 == 0 && cvb_aligned16(X) && cvb_aligned16(Y) && kind >= CVB_ACT_SILU && kind <= CVB_ACT_SIGMOID,
            "cvb_act_fwd: bad arguments");
  CVB_CUDA(cvb_launch(act_fwd_kernel, grid_for(n / 8), NT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(X), static_cast<bf16*>(Y), n / 8, kind));
  return 0;
}
extern "C" int cvb_act_bwd(const void* DY, const void* X, void* DX, int64_t n, int kind, cvb_stream_t stream) {
  CVB_CHECK(DY && X && DX && n > 0 && n % 8 == 0 && cvb_aligned16(DY) && cvb_aligned16(X) && cvb_aligned16(DX) && kind >= CVB_ACT_SILU &&
                kind <= CVB_ACT_SIGMOID,
            "cvb_act_bwd: bad arguments");
  CVB_CUDA(cvb_launch(act_bwd_kernel, grid_for(n / 8), NT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(DY), static_cast<const bf16*>(X),
                      static_cast<bf16*>(DX), n / 8, kind));
  return 0;
}

extern "C" int cvb_ln_stats(const void* X, int ldx, int64_t M, int C, float eps, float* mean, float* rstd, cvb_stream_t stream) {
  CVB_CHECK(X && mean && rstd && M > 0 && C > 0 && C % 8 == 0 && ldx % 8 == 0 && cvb_aligned16(X), "cvb_ln_stats: bad arguments");
  const int rows_per_cta = NT / 32;
  CVB_CUDA(cvb_launch(ln_stats_kernel, (unsigned)((M + rows_per_cta - 1) / rows_per_cta), NT, 0, static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(X), ldx, M, C, eps, mean, rstd));
  return 0;
}

extern "C" int cvb_gn_bwd_apply(const void* G, const void* X, const float* mean, const float* rstd, const double* sg, const double* sgx, double count,
                                const void* DRES, void* DX, int B, int rows_per_sample, int C, double* col_sum, cvb_stream_t stream) {
  CVB_CHECK(G && X && mean && rstd && sg && sgx && DX && B > 0 && rows_per_sample > 0 && C > 0 && C % 8 == 0 && C <= 2048,
            "cvb_gn_bwd_apply: bad arguments");
  int64_t M = (int64_t)B * rows_per_sample;
  RowGeom g = row_geom(M, C);
  CVB_CUDA(cvb_launch(gn_bwd_apply_kernel, g.ctas, g.nthreads, col_sum ? g.rpp * C * sizeof(float) : 0, static_cast<cudaStream_t>(stream),
      static_cast<const bf16*>(G), static_cast<const bf16*>(X), mean, rstd, sg, sgx, count, static_cast<const bf16*>(DRES), static_cast<bf16*>(DX), M,
      rows_per_sample, C, col_sum, g.cgs, g.rpp, g.rows_per_cta, static_cast<const float*>(nullptr)));
  return 0;
}

extern "C" int cvb_gn_bwd(const void* V, const void* X, const float* mean, const float* rstd, const float* gamma, double count, const void* DRES,
                          void* DX, int B, int rows_per_sample, int C, double* dgamma, double* dbeta, double* samp_ws, cvb_stream_t stream) {
  CVB_CHECK(V && X && mean && rstd && gamma && DX && dgamma && dbeta && samp_ws && B > 0 && rows_per_sample > 0 && C > 0 && C % 8 == 0 && C <= 2048,
            "cvb_gn_bwd: bad arguments");
  int64_t M = (int64_t)B * rows_per_sample;
  RowGeom g1 = row_geom(rows_per_sample, C);
  int chunks = g1.ctas;
  const int cap = (6 * cvb_num_sms() + B - 1) / B;
  int rows_per_cta = g1.rows_per_cta;
  if (chunks > cap) { rows_per_cta = ((rows_per_sample + cap - 1) / cap + g1.rpp - 1) / g1.rpp * g1.rpp; chunks = (rows_per_sample + rows_per_cta - 1) / rows_per_cta; }
  // whole warps: the per-sample sums are warp-shuffle reductions over every lane (cgs * rpp is 240..256 for C = 24, 40, 80, 96, 192, ...);
  // the threads past cgs * rpp have rr >= rpp and contribute zeros
  const int nthreads1 = (g1.nthreads + 31) / 32 * 32;
  CVB_CUDA(cvb_launch(gn_bwd_stats_kernel, dim3(chunks, B), nthreads1, 2 * C * sizeof(double), static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(V), static_cast<const bf16*>(X), mean, rstd, gamma, rows_per_sample, C, g1.cgs, g1.rpp, rows_per_cta, dgamma,
                      dbeta, samp_ws, samp_ws + B));
  RowGeom g = row_geom(M, C);
  CVB_CUDA(cvb_launch(gn_bwd_apply_kernel, g.ctas, g.nthreads, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(V),
                      static_cast<const bf16*>(X), mean, rstd, static_cast<const double*>(samp_ws), static_cast<const double*>(samp_ws + B), count,
                      static_cast<const bf16*>(DRES), static_cast<bf16*>(DX), M, rows_per_sample, C, static_cast<double*>(nullptr), g.cgs, g.rpp,
                      g.rows_per_cta, gamma));
  return 0;
}

extern "C" int cvb_global_pool_fwd(const void* X, int B, int HW, int C, void* OUT, cvb_stream_t stream) {
  CVB_CHECK(X && OUT && B > 0 && HW > 0 && C > 0 && C % 8 == 0, "cvb_global_pool_fwd: bad arguments");
  const int nc = C < CH_CHUNK ? C : CH_CHUNK;
  int cgs = nc / 8;
  int rpp = NT / cgs; if (rpp < 1) rpp = 1;
  CVB_CUDA(cvb_launch(pool_fwd_kernel, dim3(B, (C + CH_CHUNK - 1) / CH_CHUNK), cgs * rpp, nc * sizeof(double), static_cast<cudaStream_t>(stream),
                      static_cast<const bf16*>(X), HW, C, static_cast<bf16*>(OUT)));
  return 0;
}

extern "C" int cvb_global_pool_bwd(const void* DOUT, int B, int HW, int C, void* DX, cvb_stream_t stream) {
  CVB_CHECK(DOUT && DX && B > 0 && HW > 0 && C > 0 && C % 8 == 0, "cvb_global_pool_bwd: bad arguments");
  int64_t nvec = (int64_t)B * HW * (C / 8);
  CVB_CUDA(cvb_launch(pool_bwd_kernel, grid_for(nvec), NT, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(DOUT), HW, C, static_cast<bf16*>(DX), nvec));
  return 0;
}

extern "C" int cvb_stem_im2col(const float* X, int64_t sxn, int64_t sxc, int64_t sxh, int64_t sxw, int B, int H, int W, void* A, const float* mix,
                               cvb_stream_t stream) {
  CVB_CHECK(X && A && B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "cvb_stem_im2col: bad arguments (H, W must be even)");
  int64_t total = (int64_t)B * (H / 2) * (W / 2) * 4;
  CVB_CUDA(cvb_launch(stem_im2col_kernel, grid_for(total), NT, 0, static_cast<cudaStream_t>(stream), X, sxn, sxc, sxh, sxw, B, H, W, static_cast<bf16*>(A),
                      mix));
  return 0;
}

extern "C" int cvb_prep_weights(const cvb_prep_desc* descs_device, int n_desc, int max_elems, cvb_stream_t stream) {
  CVB_CHECK(descs_device && n_desc > 0 && max_elems > 0, "cvb_prep_weights: bad arguments");
  int gx = (max_elems + NT * 4 - 1) / (NT * 4);
  if (gx < 1) gx = 1;
  if (gx > 64) gx = 64;
  dim3 grid(gx, n_desc);
  CVB_CUDA(cvb_launch(prep_weights_kernel, grid, NT, 0, static_cast<cudaStream_t>(stream), descs_device));
  return 0;
}

extern "C" int cvb_unprep_grad(const float* src, float* dst, int rows, int cols, int lds, int kind, int rot, cvb_stream_t stream) {
  CVB_CHECK(src && dst && rows > 0 && cols > 0, "cvb_unprep_grad: bad arguments");
  CVB_CUDA(cvb_launch(unprep_grad_kernel, grid_for((int64_t)rows * cols), NT, 0, static_cast<cudaStream_t>(stream), src, dst, rows, cols, lds, kind, rot));
  return 0;
}
