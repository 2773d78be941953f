// Depthwise KxK convolution (K = 3 | 5, pad (K-1)/2, stride 1|2), NHWC bf16, forward and fused backward (sm_90a).
//
// HBM-bound stencils whose first implementation was instruction-issue bound (~85 instructions per element).  This version is
// built around the instruction count:
//   * a warp spans the CTA's 64 channels (lane = channel pair, one 4-byte bf16x2 access per lane = one conflict-free 128-byte
//     shared-memory wavefront per warp) and WALKS along a strip of pixels, keeping the KxK neighbourhood of the strip's rows in
//     registers (sliding window: each neighbour is loaded (R+K-1)/R times instead of K*K);
//   * all arithmetic is fp32 on channel pairs (ffma2 / fmul2 helpers), weights / dW accumulators / BN statistics stay in
//     registers for the whole batch loop of the CTA;
//   * backward: for every INPUT pixel p the same neighbourhood dy[p - tap] feeds both products,
//         dX[p] = sum_t W[t] * dy[p - t]        dW[t] += act(x[p]) * dy[p - t],
//     so one walk produces the input gradient, the weight gradient, the producer's activation backward and its BN-backward
//     statistics; x needs no halo and is read exactly once;
//   * tiles (+ zero-filled halos = the conv padding) are staged by TMA into two buffer sets with mbarriers, the next image's tiles
//     are in flight while the current one is processed.
#include "common.cuh"
#include <type_traits>

namespace {

constexpr int CB = 64;    // channels per CTA (32 lanes x channel pair)
constexpr int NT = 256;   // forward: 8 warps, 2 CTAs / SM
constexpr int SEG = 8;    // pixels a warp walks per strip (fully unrolled: the window shift is register renaming)
// backward: 16 warps for 3x3; 5x5 keeps 25 weights + 25 dW accumulators + a 6 x 5 window per lane, which needs the 255-register
// budget of 8 warps
template <int K> constexpr int bwd_threads() { return K == 3 ? 512 : 256; }
// opt-in dynamic shared memory of the backward; with the static part (5x5: 12.5 KB of fp64 dW partials) it must stay within 227 KB per CTA
template <int K> constexpr int bwd_smem_cap() { return K == 3 ? 216 * 1024 : 200 * 1024; }

// bf16x2 -> two fp32 (exact): two integer-pipe instructions, no conversion unit
__device__ __forceinline__ float2 up2(uint32_t u) { return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u)); }
__device__ __forceinline__ float2 lds2(const uint8_t* tile, int pix, int lane) {
  return up2(*reinterpret_cast<const uint32_t*>(tile + pix * 128 + lane * 4));
}

// in-place producer transform of a staged tile, 16-byte chunks: a = act(scale * x + shift) for in-bounds pixels; the zero-filled
// halo / out-of-range channels stay zero (the padding acts on the activated tensor).  s_par: [2][64] scale, shift.
template <int XMODE, int NTHR>
__device__ __forceinline__ void transform_tile(uint8_t* tile, int TH_, int TW_, int h_base, int w_base, int H, int W, int c0, int C,
                                               const float* s_par, int warp, int lane) {
  const int pch = lane & 7;
  const int lc = c0 + (pch << 3);
  if (lc >= C) return;
  float sc[8], sh[8];
  *reinterpret_cast<float4*>(sc) = *reinterpret_cast<const float4*>(s_par + pch * 8);
  *reinterpret_cast<float4*>(sc + 4) = *reinterpret_cast<const float4*>(s_par + pch * 8 + 4);
  *reinterpret_cast<float4*>(sh) = *reinterpret_cast<const float4*>(s_par + CB + pch * 8);
  *reinterpret_cast<float4*>(sh + 4) = *reinterpret_cast<const float4*>(s_par + CB + pch * 8 + 4);
  if (XMODE == CVB_A_AFF_SILU) {  // silu(z) = h + h * tanh(h), h = z / 2: fold the 1/2 into the affine parameters
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] *= 0.5f; sh[j] *= 0.5f; }
  }
  for (int ih = warp; ih < TH_; ih += NTHR / 32) {
    const int h = h_base + ih;
    if (h < 0 || h >= H) continue;
    for (int jw = lane >> 3; jw < TW_; jw += 4) {
      const int w = w_base + jw;
      if (w < 0 || w >= W) continue;
      uint4* ptr = reinterpret_cast<uint4*>(tile + (ih * TW_ + jw) * 128 + (pch << 4));
      const uint4 raw = *ptr;
      const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
      uint32_t ow[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // fp32 channel pairs: 2 ffma2 + 2 MUFU per channel pair
        float2 z = ffma2(make_float2(sc[2 * j], sc[2 * j + 1]), up2(rw[j]), make_float2(sh[2 * j], sh[2 * j + 1]));
        if (XMODE == CVB_A_AFF_SILU) z = ffma2(z, make_float2(tanh_approx_f(z.x), tanh_approx_f(z.y)), z);
        ow[j] = pack_bf162(z.x, z.y);
      }
      *ptr = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------- forward
// Output tile TH x TW, input tile IH x IW = ((TH-1)S+K) x ((TW-1)S+K) with origin (S*oh0 - P, S*ow0 - P), P = (K-1)/2.
//   stride 1: strip = 2 output rows x SEG columns, window (K+1) x K;  stride 2: strip = 1 output row x SEG columns, window K x K.
template <int XMODE, int S, int K>
__global__ void __launch_bounds__(NT, 2) dw_fwd_kernel(const __grid_constant__ CUtensorMap tmX, const cvb_dw_fwd_args p, int Ho, int Wo, int TH,
                                                       int TW, int tiles_w, int buf_bytes) {
  constexpr int P = (K - 1) / 2;
  constexpr int R = (S == 1) ? 2 : 1;
  constexpr int WR = R + K - 1;  // window rows
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ double s_cs[CB], s_cq[CB];  // fp64: the warps' fp32 partials sum exactly, whatever their order
  __shared__ __align__(16) float s_xp[2 * CB];
  __shared__ __align__(8) uint64_t bar[2];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int th_i = blockIdx.x / tiles_w, tw_i = blockIdx.x % tiles_w;
  const int oh0 = th_i * TH, ow0 = tw_i * TW;
  const int c0 = blockIdx.y * CB;
  const int IH = (TH - 1) * S + K, IW = (TW - 1) * S + K;
  const int h_base = oh0 * S - P, w_base = ow0 * S - P;
  const uint32_t tile_bytes = (uint32_t)IH * IW * 128;
  const int n_img = (p.B - (int)blockIdx.z + (int)gridDim.z - 1) / (int)gridDim.z;

  if (tid < CB) { s_cs[tid] = 0.0; s_cq[tid] = 0.0; }
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  if (tid == 0) {
    for (int i = 0; i < 2 && i < n_img; ++i) {
      mbar_expect_tx(&bar[i], tile_bytes);
      tma_load_4d(smem + i * buf_bytes, &tmX, &bar[i], c0, w_base, h_base, (int)blockIdx.z + i * (int)gridDim.z);
    }
  }
  if (XMODE != CVB_A_RAW && tid < CB) {
    const bool ok = c0 + tid < p.C;
    s_xp[tid] = ok ? __ldg(p.x_p0 + c0 + tid) : 1.f;
    s_xp[CB + tid] = ok ? __ldg(p.x_p1 + c0 + tid) : 0.f;
  }
  const int cl = c0 + 2 * lane;  // this lane's channel pair
  const bool lane_ok = cl < p.C;
  float2 wv[K * K];
#pragma unroll
  for (int t = 0; t < K * K; ++t) wv[t] = lane_ok ? make_float2(p.Wt[t * p.C + cl], p.Wt[t * p.C + cl + 1]) : make_float2(0.f, 0.f);
  float2 cs = make_float2(0.f, 0.f), cq = make_float2(0.f, 0.f);
  const int strips_w = TW / SEG;
  const int n_strips = (TH / R) * strips_w;
  const bool interior = (oh0 + TH <= Ho) && (ow0 + TW <= Wo) && (c0 + CB <= p.C);  // uniform per CTA
  __syncthreads();  // s_xp visible

  for (int i = 0; i < n_img; ++i) {
    const int b = (int)blockIdx.z + i * (int)gridDim.z;
    uint8_t* tile = smem + (i & 1) * buf_bytes;
    mbar_wait(&bar[i & 1], (i >> 1) & 1);
    if (XMODE != CVB_A_RAW) {
      transform_tile<XMODE, NT>(tile, IH, IW, h_base, w_base, p.H, p.W, c0, p.C, s_xp, warp, lane);
      __syncthreads();
    }
    bf16* __restrict__ Y = static_cast<bf16*>(p.Y) + (size_t)b * Ho * Wo * p.C + cl;
    // interior tiles (every output pixel and channel of the tile exists): no per-pixel predicates, statistics straight from the fp32
    // accumulators (the rounding error of the stored bf16 averages out over the >= 10^5 values per channel, as in the wgmma GEMM epilogue)
    auto strips = [&](auto interior_tag) {
    constexpr bool INTERIOR = decltype(interior_tag)::value;
    for (int st = warp; st < n_strips; st += NT / 32) {
      const int orow = (st / strips_w) * R, ocol = (st % strips_w) * SEG;  // tile-local output origin of the strip
      const int irow = orow * S, icol = ocol * S;                         // tile-local input origin (halo included)
      bf16* yrow[R];
#pragma unroll
      for (int r = 0; r < R; ++r) yrow[r] = Y + ((size_t)(oh0 + orow + r) * Wo + ow0 + ocol) * p.C;
      float2 win[WR][K];  // win[k][c] = input column icol + S*x + c of row irow + k
      if (S == 1) {
#pragma unroll
        for (int k = 0; k < WR; ++k)
#pragma unroll
          for (int c = 1; c < K; ++c) win[k][c] = lds2(tile, (irow + k) * IW + icol + c - 1, lane);
      } else {
#pragma unroll
        for (int k = 0; k < WR; ++k)
#pragma unroll
          for (int c = 2; c < K; ++c) win[k][c] = lds2(tile, (irow + k) * IW + icol + c - 2, lane);
      }
#pragma unroll
      for (int x = 0; x < SEG; ++x) {
        if (S == 1) {
#pragma unroll
          for (int k = 0; k < WR; ++k) {
#pragma unroll
            for (int c = 0; c < K - 1; ++c) win[k][c] = win[k][c + 1];
            win[k][K - 1] = lds2(tile, (irow + k) * IW + icol + x + K - 1, lane);
          }
        } else {
#pragma unroll
          for (int k = 0; k < WR; ++k) {
#pragma unroll
            for (int c = 0; c < K - 2; ++c) win[k][c] = win[k][c + 2];
            win[k][K - 2] = lds2(tile, (irow + k) * IW + icol + 2 * x + K - 2, lane);
            win[k][K - 1] = lds2(tile, (irow + k) * IW + icol + 2 * x + K - 1, lane);
          }
        }
        const int gw = ow0 + ocol + x;
#pragma unroll
        for (int r = 0; r < R; ++r) {
          float2 acc = make_float2(0.f, 0.f);
#pragma unroll
          for (int u = 0; u < K; ++u)
#pragma unroll
            for (int v = 0; v < K; ++v) acc = ffma2(wv[u * K + v], win[r + u][v], acc);
          const uint32_t pk = pack_bf162(acc.x, acc.y);
          if (INTERIOR) {
            cs = fadd2(cs, acc);
            cq = ffma2(acc, acc, cq);
            *reinterpret_cast<uint32_t*>(yrow[r]) = pk;
          } else {
            const bool ok = (oh0 + orow + r < Ho) && (gw < Wo) && lane_ok;
            float2 rv = up2(pk);  // branch-free, only the store is predicated
            rv.x = ok ? rv.x : 0.f;
            rv.y = ok ? rv.y : 0.f;
            cs = fadd2(cs, rv);
            cq = ffma2(rv, rv, cq);
            if (ok) *reinterpret_cast<uint32_t*>(yrow[r]) = pk;
          }
          yrow[r] += p.C;
        }
      }
    }
    };
    if (interior) strips(std::true_type{}); else strips(std::false_type{});
    __syncthreads();  // every thread is done with this buffer
    if (tid == 0 && i + 2 < n_img) {
      fence_proxy_async();  // order the generic-proxy accesses above before the async-proxy overwrite
      mbar_expect_tx(&bar[i & 1], tile_bytes);
      tma_load_4d(tile, &tmX, &bar[i & 1], c0, w_base, h_base, (int)blockIdx.z + (i + 2) * (int)gridDim.z);
    }
  }
  if (p.col_sum) {
    if (lane_ok) {
      atomicAdd(&s_cs[2 * lane], (double)cs.x); atomicAdd(&s_cs[2 * lane + 1], (double)cs.y);
      atomicAdd(&s_cq[2 * lane], (double)cq.x); atomicAdd(&s_cq[2 * lane + 1], (double)cq.y);
    }
    __syncthreads();
    if (tid < CB && c0 + tid < p.C) {
      atomicAdd(p.col_sum + c0 + tid, s_cs[tid]);
      atomicAdd(p.col_sq + c0 + tid, s_cq[tid]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ backward
// Per image tile: (dz, x) double-buffered, y2 single-buffered (it is consumed by step 1 only and refilled right after it).
//   1. dy = c1*dz + c2*y2 + c3 in place (in-bounds pixels only: the zero halo is the transposed conv's padding)
//   2. one walk over the tile's INPUT pixels: dX, dW, activation backward, BN-backward statistics of the producer.
// stride 1: strip = 2 input rows x SEG columns, dy window (K+1) x K (halo origin -P).
// stride 2: strip = 1 OUTPUT row x SEG output columns = 2 x 2SEG input pixels.  Input pixel (2i+a, 2j+b) receives tap (u, v) from
//   dy[i + (a+P-u)/2, j + (b+P-v)/2] when a+P-u and b+P-v are even, so the dy rows / columns it needs are i-LO .. i+1 with LO = P/2:
//   dy window (LO+2) x (LO+2), halo LO on the low side and 1 on the high side.  3x3 (LO = 0):
//   x(2i,2j)     <- W11 dy[i,j]                      x(2i,2j+1)   <- W10 dy[i,j+1] + W12 dy[i,j]
//   x(2i+1,2j)   <- W01 dy[i+1,j] + W21 dy[i,j]      x(2i+1,2j+1) <- W00 dy[i+1,j+1] + W02 dy[i+1,j] + W20 dy[i,j+1] + W22 dy[i,j]
struct PixOut {
  float2 a;     // act(BN(x)) (dW operand)
  float2 dact;  // d act / d z
  float2 xr;    // raw x (statistics operand)
};
template <int XMODE>
__device__ __forceinline__ PixOut load_x(const uint8_t* sX, int pix, int lane, float2 xsc, float2 xsh, bool ok) {
  PixOut o;
  o.xr = lds2(sX, pix, lane);
  if (XMODE == CVB_A_RAW) {
    o.a = o.xr;
    o.dact = make_float2(1.f, 1.f);
  } else {
    const float2 z = ffma2(xsc, o.xr, xsh);
    if (XMODE == CVB_A_AFF_SILU) {
      // one sigmoid per element serves both uses: a = z*s and silu'(z) = s + a*(1-s)
      const float sx = sigmoid_f(z.x), sy = sigmoid_f(z.y);
      o.a = make_float2(z.x * sx, z.y * sy);
      o.dact = make_float2(fmaf(o.a.x, 1.0f - sx, sx), fmaf(o.a.y, 1.0f - sy, sy));
    } else {
      o.a = z;
      o.dact = make_float2(1.f, 1.f);
    }
  }
  if (!ok) o.a = make_float2(0.f, 0.f);  // pixels past the image edge must not reach dW
  return o;
}
template <int XMODE, bool INTERIOR>
__device__ __forceinline__ void finish_pixel(float2 d, const PixOut& o, float2& cs, float2& cq, bf16* dst, bool ok) {
  if (XMODE == CVB_A_AFF_SILU) d = fmul2(d, o.dact);
  const uint32_t pk = pack_bf162(d.x, d.y);
  if (INTERIOR) {  // whole tile inside the image: no predicates; statistics from the fp32 values (rounding averages out over the channel)
    if (XMODE != CVB_A_RAW) {
      cs = fadd2(cs, d);
      cq = ffma2(d, o.xr, cq);
    }
    *reinterpret_cast<uint32_t*>(dst) = pk;
    return;
  }
  // branch-free: out-of-image pixels / channels contribute zeros to the statistics and only the store is predicated
  if (XMODE != CVB_A_RAW) {
    float2 rv = up2(pk);
    rv.x = ok ? rv.x : 0.f;
    rv.y = ok ? rv.y : 0.f;
    cs = fadd2(cs, rv);
    cq = ffma2(rv, o.xr, cq);
  }
  if (ok) *reinterpret_cast<uint32_t*>(dst) = pk;
}

template <int GMODE, int XMODE, int S, int K>
__global__ void __launch_bounds__(bwd_threads<K>(), 1) dw_bwd_kernel(const __grid_constant__ CUtensorMap tmDZ, const __grid_constant__ CUtensorMap tmY2,
                                                                     const __grid_constant__ CUtensorMap tmX, const cvb_dw_bwd_args p, int Ho, int Wo,
                                                                     int TH, int TW, int tiles_w, int g_bytes, int x_bytes) {
  constexpr bool BNB = (GMODE == CVB_A_BNB);
  constexpr int NTB = bwd_threads<K>();
  constexpr int P = (K - 1) / 2, LO = P / 2;
  constexpr int GLO = (S == 1) ? P : LO, GHI = (S == 1) ? P : 1;  // dy halo below / above the tile
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ double s_cs[CB], s_cq[CB];  // fp64: the warps' fp32 partials sum exactly, whatever their order
  __shared__ double s_dw[K * K][CB];
  __shared__ __align__(16) float s_gp[3 * CB];
  __shared__ __align__(8) uint64_t bar[2], ybar;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int th_i = blockIdx.x / tiles_w, tw_i = blockIdx.x % tiles_w;
  const int oh0 = th_i * TH, ow0 = tw_i * TW;
  const int c0 = blockIdx.y * CB;
  const int GH = TH + GLO + GHI, GW = TW + GLO + GHI;
  const int XH = S * TH, XW = S * TW;  // input tile, no halo
  const int gh_base = oh0 - GLO, gw_base = ow0 - GLO;
  const int xh_base = S * oh0, xw_base = S * ow0;
  const int set_bytes = g_bytes + x_bytes;
  uint8_t* sY2 = smem + 2 * set_bytes;
  const uint32_t g_tx = (uint32_t)GH * GW * 128, x_tx = (uint32_t)XH * XW * 128;
  const int n_img = (p.B - (int)blockIdx.z + (int)gridDim.z - 1) / (int)gridDim.z;

  auto issue = [&](int i) {  // one elected thread: (dz, x) of the CTA's i-th image into set i & 1
    uint8_t* base = smem + (i & 1) * set_bytes;
    const int b = (int)blockIdx.z + i * (int)gridDim.z;
    mbar_expect_tx(&bar[i & 1], g_tx + x_tx);
    tma_load_4d(base, &tmDZ, &bar[i & 1], c0, gw_base, gh_base, b);
    tma_load_4d(base + g_bytes, &tmX, &bar[i & 1], c0, xw_base, xh_base, b);
  };
  auto issue_y2 = [&](int i) {
    mbar_expect_tx(&ybar, g_tx);
    tma_load_4d(sY2, &tmY2, &ybar, c0, gw_base, gh_base, (int)blockIdx.z + i * (int)gridDim.z);
  };

  for (int i = tid; i < K * K * CB; i += NTB) (&s_dw[0][0])[i] = 0.0;
  if (tid < CB) { s_cs[tid] = 0.0; s_cq[tid] = 0.0; }
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_init(&ybar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  if (tid == 0) {
    for (int i = 0; i < 2 && i < n_img; ++i) issue(i);
    if (BNB) issue_y2(0);
  }
  if (BNB && tid < CB) {
    const bool ok = c0 + tid < p.C;
    s_gp[tid] = ok ? __ldg(p.g_p0 + c0 + tid) : 0.f;
    s_gp[CB + tid] = ok ? __ldg(p.g_p1 + c0 + tid) : 0.f;
    s_gp[2 * CB + tid] = ok ? __ldg(p.g_p2 + c0 + tid) : 0.f;
  }
  const int cl = c0 + 2 * lane;
  const bool lane_ok = cl < p.C;
  float2 wv[K * K], accw[K * K];
#pragma unroll
  for (int t = 0; t < K * K; ++t) {
    wv[t] = lane_ok ? make_float2(p.Wt[t * p.C + cl], p.Wt[t * p.C + cl + 1]) : make_float2(0.f, 0.f);
    accw[t] = make_float2(0.f, 0.f);
  }
  float2 xsc = make_float2(1.f, 1.f), xsh = make_float2(0.f, 0.f);
  if (XMODE != CVB_A_RAW && lane_ok) {
    xsc = make_float2(__ldg(p.x_p0 + cl), __ldg(p.x_p0 + cl + 1));
    xsh = make_float2(__ldg(p.x_p1 + cl), __ldg(p.x_p1 + cl + 1));
  }
  float2 cs = make_float2(0.f, 0.f), cq = make_float2(0.f, 0.f);
  const int strips_w = TW / SEG;
  const int n_strips = (S == 1 ? TH / 2 : TH) * strips_w;
  const bool interior = (xh_base + XH <= p.H) && (xw_base + XW <= p.W) && (c0 + CB <= p.C);  // uniform per CTA: the whole input tile exists
  __syncthreads();  // s_gp visible

  for (int i = 0; i < n_img; ++i) {
    const int b = (int)blockIdx.z + i * (int)gridDim.z;
    uint8_t* sG = smem + (i & 1) * set_bytes;
    const uint8_t* sX = sG + g_bytes;
    mbar_wait(&bar[i & 1], (i >> 1) & 1);
    // ---- 1. dy = c1*dz + c2*y2 + c3, in place, in-bounds pixels only
    if (BNB) {
      mbar_wait(&ybar, i & 1);
      const int pch = lane & 7;
      if (c0 + (pch << 3) < p.C) {
        float g0[8], g1[8], g2[8];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          *reinterpret_cast<float4*>(g0 + 4 * q) = *reinterpret_cast<const float4*>(s_gp + pch * 8 + 4 * q);
          *reinterpret_cast<float4*>(g1 + 4 * q) = *reinterpret_cast<const float4*>(s_gp + CB + pch * 8 + 4 * q);
          *reinterpret_cast<float4*>(g2 + 4 * q) = *reinterpret_cast<const float4*>(s_gp + 2 * CB + pch * 8 + 4 * q);
        }
        for (int gi = warp; gi < GH; gi += NTB / 32) {
          const int oh = gh_base + gi;
          if (oh < 0 || oh >= Ho) continue;
          for (int gj = lane >> 3; gj < GW; gj += 4) {
            const int ow = gw_base + gj;
            if (ow < 0 || ow >= Wo) continue;
            const int off = (gi * GW + gj) * 128 + (pch << 4);
            uint4* pz = reinterpret_cast<uint4*>(sG + off);
            const uint4 zr = *pz, yr = *reinterpret_cast<const uint4*>(sY2 + off);
            const uint32_t zw[4] = {zr.x, zr.y, zr.z, zr.w}, yw[4] = {yr.x, yr.y, yr.z, yr.w};
            uint32_t o4[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {  // packed fp32 pairs
              const float2 t = ffma2(make_float2(g1[2 * j], g1[2 * j + 1]), up2(yw[j]), make_float2(g2[2 * j], g2[2 * j + 1]));
              const float2 v = ffma2(make_float2(g0[2 * j], g0[2 * j + 1]), up2(zw[j]), t);
              o4[j] = pack_bf162(v.x, v.y);
            }
            *pz = make_uint4(o4[0], o4[1], o4[2], o4[3]);
          }
        }
      }
      __syncthreads();
      if (tid == 0 && i + 1 < n_img) {
        fence_proxy_async();
        issue_y2(i + 1);
      }
    }
    // ---- 2. the walk
    bf16* __restrict__ DX = static_cast<bf16*>(p.DX) + (size_t)b * p.H * p.W * p.C + cl;
    auto strips = [&](auto interior_tag) {
    constexpr bool INTERIOR = decltype(interior_tag)::value;
    for (int st = warp; st < n_strips; st += NTB / 32) {
      const int scol = (st % strips_w) * SEG;
      if (S == 1) {
        const int r0 = (st / strips_w) * 2;  // tile-local input rows r0, r0+1; dy halo rows r0 .. r0+K, halo cols scol .. scol+SEG+K-2
        bf16* dxrow[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) dxrow[r] = DX + ((size_t)(oh0 + r0 + r) * p.W + ow0 + scol) * p.C;
        float2 win[K + 1][K];
#pragma unroll
        for (int k = 0; k < K + 1; ++k)
#pragma unroll
          for (int c = 1; c < K; ++c) win[k][c] = lds2(sG, (r0 + k) * GW + scol + c - 1, lane);
#pragma unroll
        for (int x = 0; x < SEG; ++x) {
#pragma unroll
          for (int k = 0; k < K + 1; ++k) {
#pragma unroll
            for (int c = 0; c < K - 1; ++c) win[k][c] = win[k][c + 1];
            win[k][K - 1] = lds2(sG, (r0 + k) * GW + scol + x + K - 1, lane);
          }
          const int w = ow0 + scol + x;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int h = oh0 + r0 + r;
            const bool ok = INTERIOR || ((h < p.H) && (w < p.W) && lane_ok);
            const PixOut o = load_x<XMODE>(sX, (r0 + r) * XW + scol + x, lane, xsc, xsh, ok);
            float2 d = make_float2(0.f, 0.f);
            // dyn[u][v] = dy[h+P-u][w+P-v] = win[r+K-1-u][K-1-v]
#pragma unroll
            for (int u = 0; u < K; ++u)
#pragma unroll
              for (int v = 0; v < K; ++v) {
                d = ffma2(wv[u * K + v], win[r + K - 1 - u][K - 1 - v], d);
                accw[u * K + v] = ffma2(o.a, win[r + K - 1 - u][K - 1 - v], accw[u * K + v]);
              }
            finish_pixel<XMODE, INTERIOR>(d, o, cs, cq, dxrow[r], ok);
            dxrow[r] += p.C;
          }
        }
      } else {
        constexpr int NW = LO + 2;     // win[k][c] = dy[i - LO + k][j - LO + c]
        const int i0 = st / strips_w;  // tile-local output row i - oh0; dy tile rows i0 .. i0+LO+1; input rows 2*i0, 2*i0+1
        bf16* dxrow0 = DX + ((size_t)(2 * (oh0 + i0)) * p.W + 2 * (ow0 + scol)) * p.C;
        float2 win[NW][NW];
#pragma unroll
        for (int k = 0; k < NW; ++k)
#pragma unroll
          for (int c = 1; c < NW; ++c) win[k][c] = lds2(sG, (i0 + k) * GW + scol + c - 1, lane);
#pragma unroll
        for (int x = 0; x < SEG; ++x) {
#pragma unroll
          for (int k = 0; k < NW; ++k) {
#pragma unroll
            for (int c = 0; c < NW - 1; ++c) win[k][c] = win[k][c + 1];
            win[k][NW - 1] = lds2(sG, (i0 + k) * GW + scol + x + NW - 1, lane);
          }
          const int hh = 2 * (oh0 + i0), ww = 2 * (ow0 + scol + x);
          const int xp = (2 * i0) * XW + 2 * (scol + x);
          bf16* dx0 = dxrow0 + (size_t)(2 * x) * p.C;
#pragma unroll
          for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b) {  // input pixel (2i+a, 2j+b)
              const bool ok = INTERIOR || ((hh + a < p.H) && (ww + b < p.W) && lane_ok);
              const PixOut o = load_x<XMODE>(sX, xp + a * XW + b, lane, xsc, xsh, ok);
              float2 d = make_float2(0.f, 0.f);
              bool first = true;  // (resolved at compile time) the first product is a plain multiply
#pragma unroll
              for (int u = 0; u < K; ++u) {
                if ((a + P - u) & 1) continue;
#pragma unroll
                for (int v = 0; v < K; ++v) {
                  if ((b + P - v) & 1) continue;
                  const float2 g = win[(a + P - u) / 2 + LO][(b + P - v) / 2 + LO];
                  d = first ? fmul2(wv[u * K + v], g) : ffma2(wv[u * K + v], g, d);
                  first = false;
                  accw[u * K + v] = ffma2(o.a, g, accw[u * K + v]);
                }
              }
              finish_pixel<XMODE, INTERIOR>(d, o, cs, cq, dx0 + (size_t)a * p.W * p.C + b * p.C, ok);
            }
        }
      }
    }
    };
    if (interior) strips(std::true_type{}); else strips(std::false_type{});
    __syncthreads();  // every thread is done with this buffer set
    if (tid == 0 && i + 2 < n_img) {
      fence_proxy_async();
      issue(i + 2);
    }
  }

  // ---- reductions (once per CTA)
  if (lane_ok) {
#pragma unroll
    for (int t = 0; t < K * K; ++t) {
      atomicAdd(&s_dw[t][2 * lane], (double)accw[t].x);
      atomicAdd(&s_dw[t][2 * lane + 1], (double)accw[t].y);
    }
    if (p.col_sum) {
      atomicAdd(&s_cs[2 * lane], (double)cs.x); atomicAdd(&s_cs[2 * lane + 1], (double)cs.y);
      atomicAdd(&s_cq[2 * lane], (double)cq.x); atomicAdd(&s_cq[2 * lane + 1], (double)cq.y);
    }
  }
  __syncthreads();
  for (int i = tid; i < K * K * CB; i += NTB) {
    int tp = i / CB, c = i % CB;
    if (c0 + c < p.C) atomicAdd(reinterpret_cast<double*>(p.dWt) + tp * p.C + c0 + c, s_dw[tp][c]);  // fp64 scratch (cvb_dw_bwd)
  }
  if (p.col_sum && tid < CB && c0 + tid < p.C) {
    atomicAdd(p.col_sum + c0 + tid, s_cs[tid]);
    atomicAdd(p.col_sq + c0 + tid, s_cq[tid]);
  }
}

int round1k(int v) { return (v + 1023) / 1024 * 1024; }

}  // namespace

int cvb_dw_fwd_dilated(const cvb_dw_fwd_args& a, cudaStream_t st);  // dwconv_dilated.cu
int cvb_dw_bwd_dilated(const cvb_dw_bwd_args& a, cudaStream_t st);

extern "C" int cvb_dw_fwd(const cvb_dw_fwd_args* args, cvb_stream_t stream) {
  CVB_CHECK(args != nullptr, "cvb_dw_fwd: null args");
  const cvb_dw_fwd_args& a = *args;
  CVB_CHECK(a.B > 0 && a.H > 0 && a.W > 0 && a.C > 0 && a.C % 8 == 0, "cvb_dw_fwd: bad shape B=%d H=%d W=%d C=%d (C %% 8 == 0)", a.B, a.H, a.W, a.C);
  CVB_CHECK(a.stride == 1 || a.stride == 2, "cvb_dw_fwd: stride must be 1 or 2");
  CVB_CHECK(a.X && a.Wt && a.Y && cvb_aligned16(a.X) && cvb_aligned16(a.Y), "cvb_dw_fwd: null / misaligned operand");
  CVB_CHECK(a.x_mode == CVB_A_RAW || ((a.x_mode == CVB_A_AFF || a.x_mode == CVB_A_AFF_SILU) && a.x_p0 && a.x_p1), "cvb_dw_fwd: bad x_mode %d", a.x_mode);
  if (a.col_sum) CVB_CHECK(a.col_sq != nullptr, "cvb_dw_fwd: col_sq missing");
  CVB_CHECK(a.dilation >= 0 && a.dilation <= 64, "cvb_dw_fwd: bad dilation %d", a.dilation);
  CVB_CHECK(a.ksize == 0 || a.ksize == 3 || a.ksize == 5, "cvb_dw_fwd: kernel size must be 3 or 5, got %d", a.ksize);
  CVB_CHECK(a.ksize != 5 || a.dilation <= 1, "cvb_dw_fwd: a dilated 5x5 kernel is not implemented");
  if (a.dilation > 1) return cvb_dw_fwd_dilated(a, static_cast<cudaStream_t>(stream));
  const int s = a.stride, K = a.ksize == 5 ? 5 : 3;
  const int Ho = (a.H - 1) / s + 1, Wo = (a.W - 1) / s + 1;
  // two CTAs per SM: two input buffers of <= ~46 KB each (5x5, stride 1: 8-row tiles keep the 20-column halo'd tile inside that)
  const int TW = (s == 1 && Wo > 8) ? 16 : 8;
  const int TH = (s == 1 && K == 3) ? (Ho > 8 ? 16 : 8) : 8;
  const int tiles_h = (Ho + TH - 1) / TH, tiles_w = (Wo + TW - 1) / TW;
  const int IH = (TH - 1) * s + K, IW = (TW - 1) * s + K;
  const int buf_bytes = round1k(IH * IW * 128);
  size_t smem = (size_t)2 * buf_bytes + 1024;
  const int cblocks = (a.C + CB - 1) / CB;
  int per_img = tiles_h * tiles_w * cblocks;
  int gz = (8 * cvb_num_sms() + per_img - 1) / per_img;  // batch loop inside the CTA: double-buffered TMA + bounded statistics atomics
  if (gz > a.B) gz = a.B;
  if (gz < 1) gz = 1;
  dim3 grid(tiles_h * tiles_w, cblocks, gz);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap tmX;
  if (cvb_make_tmap_nhwc(&tmX, a.X, a.B, a.H, a.W, a.C, IH, IW, CB, 0)) return 1;
#define CVB_DW_FWD(MODE, S, KS)                                                                                          \
  {                                                                                                                      \
    static bool attr = false;                                                                                            \
    if (!attr) { CVB_CUDA(cudaFuncSetAttribute(dw_fwd_kernel<MODE, S, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024)); attr = true; } \
    CVB_CUDA(cvb_launch(dw_fwd_kernel<MODE, S, KS>, grid, NT, smem, st, tmX, a, Ho, Wo, TH, TW, tiles_w, buf_bytes));     \
  }
#define CVB_DW_FWD_X(S, KS)                                                  \
  {                                                                          \
    if (a.x_mode == CVB_A_RAW) CVB_DW_FWD(CVB_A_RAW, S, KS)                  \
    else if (a.x_mode == CVB_A_AFF) CVB_DW_FWD(CVB_A_AFF, S, KS)             \
    else CVB_DW_FWD(CVB_A_AFF_SILU, S, KS)                                   \
  }
  if (K == 3) {
    if (s == 1) CVB_DW_FWD_X(1, 3) else CVB_DW_FWD_X(2, 3)
  } else {
    if (s == 1) CVB_DW_FWD_X(1, 5) else CVB_DW_FWD_X(2, 5)
  }
#undef CVB_DW_FWD_X
#undef CVB_DW_FWD
  CVB_LAUNCH_CHECK();
  return 0;
}

extern "C" int cvb_dw_bwd(const cvb_dw_bwd_args* args, cvb_stream_t stream) {
  CVB_CHECK(args != nullptr, "cvb_dw_bwd: null args");
  const cvb_dw_bwd_args& a = *args;
  CVB_CHECK(a.B > 0 && a.H > 0 && a.W > 0 && a.C > 0 && a.C % 8 == 0, "cvb_dw_bwd: bad shape");
  CVB_CHECK(a.stride == 1 || a.stride == 2, "cvb_dw_bwd: stride must be 1 or 2");
  CVB_CHECK(a.DZ && a.X && a.Wt && a.DX && a.dWt && cvb_aligned16(a.DZ) && cvb_aligned16(a.X) && cvb_aligned16(a.DX), "cvb_dw_bwd: null / misaligned operand");
  CVB_CHECK(a.g_mode == CVB_A_RAW || (a.g_mode == CVB_A_BNB && a.Y2 && a.g_p0 && a.g_p1 && a.g_p2), "cvb_dw_bwd: bad g_mode %d", a.g_mode);
  CVB_CHECK(a.x_mode == CVB_A_RAW || ((a.x_mode == CVB_A_AFF || a.x_mode == CVB_A_AFF_SILU) && a.x_p0 && a.x_p1), "cvb_dw_bwd: bad x_mode %d", a.x_mode);
  if (a.col_sum) CVB_CHECK(a.col_sq != nullptr, "cvb_dw_bwd: col_sq missing");
  CVB_CHECK(a.dilation >= 0 && a.dilation <= 64, "cvb_dw_bwd: bad dilation %d", a.dilation);
  CVB_CHECK(a.ksize == 0 || a.ksize == 3 || a.ksize == 5, "cvb_dw_bwd: kernel size must be 3 or 5, got %d", a.ksize);
  CVB_CHECK(a.ksize != 5 || a.dilation <= 1, "cvb_dw_bwd: a dilated 5x5 kernel is not implemented");
  if (a.dilation > 1) {
    // the dilated kernel's per-block dW partials meet in the same fp64 scratch as the walk kernels' (order-independent, so reproducible)
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* ws = nullptr;
    if (cvb_det_alloc(&ws, (size_t)9 * a.C, st)) return 2;
    cvb_dw_bwd_args b = a;
    b.dWt = reinterpret_cast<float*>(ws);
    int rc = cvb_dw_bwd_dilated(b, st);
    if (rc == 0) rc = cvb_det_add(ws, a.dWt, 9, a.C, a.C, st);
    const int rf = cvb_det_free(ws, st);
    return rc ? rc : rf;
  }
  if (a.stride == 2) CVB_CHECK(a.H % 2 == 0 && a.W % 2 == 0, "cvb_dw_bwd: stride 2 needs even H, W");
  const int s = a.stride, K = a.ksize == 5 ? 5 : 3;
  const int Ho = (a.H - 1) / s + 1, Wo = (a.W - 1) / s + 1;
  // one CTA per SM; stride 1: 16 x 16 input pixels (5x5: 8 x 16, the 4-pixel halo and the 25-tap dW scratch must fit next to the
  // double buffers), stride 2: 8 x 16 outputs = 16 x 32 input pixels (small maps: 8-wide tiles)
  const int TW = Wo > 8 ? 16 : 8;
  const int TH = (s == 1 && K == 3) ? (Ho > 8 ? 16 : 8) : 8;
  const int tiles_h = (Ho + TH - 1) / TH, tiles_w = (Wo + TW - 1) / TW;
  const int P = (K - 1) / 2, halo = (s == 1) ? 2 * P : P / 2 + 1;
  const int GH = TH + halo, GW = TW + halo;
  const int XH = s * TH, XW = s * TW;
  const int g_bytes = round1k(GH * GW * 128), x_bytes = round1k(XH * XW * 128);
  const bool bnb = (a.g_mode == CVB_A_BNB);
  size_t smem = (size_t)2 * (g_bytes + x_bytes) + (bnb ? g_bytes : 0) + 1024;
  const int cblocks = (a.C + CB - 1) / CB;
  // batch loop inside the CTA (double-buffered TMA, dW / statistics flushed once): one CTA per SM, a few waves
  int per_img = tiles_h * tiles_w * cblocks;
  int want = 4 * cvb_num_sms();
  int gz = (want + per_img - 1) / per_img;
  if (gz > a.B) gz = a.B;
  if (gz < 1) gz = 1;
  dim3 grid(tiles_h * tiles_w, cblocks, gz);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap tmDZ, tmY2, tmX;
  if (cvb_make_tmap_nhwc(&tmDZ, a.DZ, a.B, Ho, Wo, a.C, GH, GW, CB, 0)) return 1;
  if (cvb_make_tmap_nhwc(&tmY2, bnb ? a.Y2 : a.DZ, a.B, Ho, Wo, a.C, GH, GW, CB, 0)) return 1;
  if (cvb_make_tmap_nhwc(&tmX, a.X, a.B, a.H, a.W, a.C, XH, XW, CB, 0)) return 1;
  // the CTAs' dW partials meet in an fp64 scratch (order-independent), added to dWt afterwards
  double* ws = nullptr;
  if (cvb_det_alloc(&ws, (size_t)K * K * a.C, st)) return 2;
  cvb_dw_bwd_args b = a;
  b.dWt = reinterpret_cast<float*>(ws);
#define CVB_DW_BWD(GM, XM, S, KS)                                                                                        \
  {                                                                                                                      \
    static bool attr = false;                                                                                            \
    if (!attr) { CVB_CUDA(cudaFuncSetAttribute(dw_bwd_kernel<GM, XM, S, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bwd_smem_cap<KS>())); attr = true; } \
    CVB_CUDA(cvb_launch(dw_bwd_kernel<GM, XM, S, KS>, grid, bwd_threads<KS>(), smem, st, tmDZ, tmY2, tmX, b, Ho, Wo, TH, TW, tiles_w, g_bytes,   \
                        x_bytes));                                                                                       \
  }
#define CVB_DW_BWD_X(GM, S, KS)                                               \
  {                                                                          \
    if (a.x_mode == CVB_A_RAW) CVB_DW_BWD(GM, CVB_A_RAW, S, KS)               \
    else if (a.x_mode == CVB_A_AFF) CVB_DW_BWD(GM, CVB_A_AFF, S, KS)          \
    else CVB_DW_BWD(GM, CVB_A_AFF_SILU, S, KS)                                \
  }
#define CVB_DW_BWD_S(GM, KS)                                                  \
  {                                                                          \
    if (s == 1) CVB_DW_BWD_X(GM, 1, KS) else CVB_DW_BWD_X(GM, 2, KS)          \
  }
  if (K == 3) {
    if (!bnb) CVB_DW_BWD_S(CVB_A_RAW, 3) else CVB_DW_BWD_S(CVB_A_BNB, 3)
  } else {
    if (!bnb) CVB_DW_BWD_S(CVB_A_RAW, 5) else CVB_DW_BWD_S(CVB_A_BNB, 5)
  }
#undef CVB_DW_BWD_S
#undef CVB_DW_BWD_X
#undef CVB_DW_BWD
  CVB_LAUNCH_CHECK();
  if (cvb_det_add(ws, a.dWt, K * K, a.C, a.C, st)) return 2;
  return cvb_det_free(ws, st);
}
