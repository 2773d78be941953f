// wgmma / TMA weight-gradient GEMM (sm_90a):   dW[N,K] += sum_m load(G)[m,n] * load(A)[m,k],  dbias[n] += sum_m load(G)[m,n]
//
// The reduction runs over PIXELS, so both operands are "MN-major" for the tensor core: a [pixels x channels] tile with the channels
// contiguous is exactly the canonical MN-major SWIZZLE_128B layout (8 pixel rows x 128 B atoms) that TMA produces with a
// [64 channel x rows] box -- wgmma reads it transposed, no transposition anywhere.  One CTA owns a whole [128 x <=128] block of dW
// in the registers of two consumer warpgroups (64 dW rows each) and streams its slice of the pixel range through a TMA ring, so
// every activation / gradient element is read ONCE per (N-block, K-block) instead of once per 64x64 tile (the mma.sync kernel is
// L2-bandwidth bound on exactly that re-reading).  Warp roles:
//   warps 0-7   consumers     : 4 x wgmma.m64nKBk16 (K = 16 pixels each) per stage, both operands MN-major; after the last stage
//                               fp64 reductions of the accumulator registers into the dW scratch (see DetScratch)
//   warp 8      TMA producer  : per stage [64 pixels] x {G: 128 ch (+ G2 for BN-backward), A: <=128 ch}, 64-channel boxes
//   warps 9-16  transform     : in-place operand prologues in shared memory (BN-backward on G, BN+SiLU / SiLU / GroupNorm on A),
//                               bias-gradient column sums, fence.proxy.async, hand the stage to the consumers
// Split over the pixel range (grid.z) so that ~all SMs are busy; partial sums meet in dW through the fp32 reductions.
#include "common.cuh"

namespace {

constexpr int WT_BMP = 64;                 // pixels per stage
constexpr int WT_BOX = WT_BMP * 128;       // bytes of one [64 pixels x 64 channels] box (8 swizzle atoms of 1 KB)
constexpr int WT_KB = 128;                 // dW columns per CTA (at most; K = 64 layers use 64)
constexpr int WT_XF_WARPS = 8;
constexpr int WT_CONSUMERS = 256;          // two warpgroups
constexpr int WT_PRODUCER_WARP = WT_CONSUMERS / 32;
constexpr int WT_XF0 = WT_CONSUMERS + 32;  // first transform thread
constexpr int WT_THREADS = WT_XF0 + WT_XF_WARPS * 32;
constexpr int WT_MAX_STAGES = 6;

// MN-major operand, 128-byte swizzle: LBO = distance between 64-channel boxes (8 KB), SBO = distance between 8-pixel groups (1 KB)
__device__ __forceinline__ uint64_t desc_mn_sw128(uint32_t saddr) { return wgmma_desc(saddr, WT_BOX, 1024, WG_SW128); }
// byte offset of the 16-byte chunk `ch` (logical, 0..7) of pixel row `row` inside one [64 x 64ch] box (TMA SWIZZLE_128B image)
__device__ __forceinline__ uint32_t sw128(int row, int ch) { return static_cast<uint32_t>(row * 128 + ((ch ^ (row & 7)) << 4)); }

template <int GMODE, int AMODE, int KB>
__global__ void __launch_bounds__(WT_THREADS, 1)
    pw_wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmG2, const __grid_constant__ CUtensorMap tmA,
                       const cvb_wgrad_args p, int m_per_cta, int NST, int stage_bytes) {
  constexpr bool BNB = (GMODE == CVB_A_BNB);
  constexpr bool A_HAS_P = (AMODE == CVB_A_AFF || AMODE == CVB_A_AFF_SILU || AMODE == CVB_A_GN);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * 128, k0 = blockIdx.y * WT_KB;
  const int m_begin = blockIdx.z * m_per_cta;
  const int m_end = min(p.M, m_begin + m_per_cta);
  const int NS = (m_end - m_begin + WT_BMP - 1) / WT_BMP;   // >= 1 by construction of the grid
  constexpr int a_boxes = KB / 64;
  const int a_off = (BNB ? 2 : 1) * 2 * WT_BOX;             // stage layout: [G: 2 boxes][G2: 2 boxes (BNB)][A: a_boxes boxes]

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  __shared__ __align__(8) uint64_t full[WT_MAX_STAGES], ready[WT_MAX_STAGES], empty[WT_MAX_STAGES];
  __shared__ double s_db[128];

  if (tid == 0) {
    for (int i = 0; i < NST; ++i) { mbar_init(&full[i], 1); mbar_init(&ready[i], WT_XF_WARPS); mbar_init(&empty[i], 2); }
    fence_mbar_init();
  }
  if (tid < 128) s_db[tid] = 0.0;
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp == WT_PRODUCER_WARP) {
    // ===================================================== TMA producer
    if (lane == 0) {
      for (int s = 0; s < NS; ++s) {
        const int slot = s % NST;
        if (s >= NST) mbar_wait(&empty[slot], ((s / NST) - 1) & 1);
        uint8_t* st = smem + slot * stage_bytes;
        const int m = m_begin + s * WT_BMP;
        mbar_expect_tx(&full[slot], (uint32_t)stage_bytes);
        tma_load_2d(st, &tmG, &full[slot], n0, m);
        tma_load_2d(st + WT_BOX, &tmG, &full[slot], n0 + 64, m);
        if (BNB) {
          tma_load_2d(st + 2 * WT_BOX, &tmG2, &full[slot], n0, m);
          tma_load_2d(st + 3 * WT_BOX, &tmG2, &full[slot], n0 + 64, m);
        }
        for (int bx = 0; bx < a_boxes; ++bx) tma_load_2d(st + a_off + bx * WT_BOX, &tmA, &full[slot], k0 + bx * 64, m);
      }
    }
  } else if (warp < WT_PRODUCER_WARP) {
    // ===================================================== consumers: dW rows [64 wg, 64 wg + 64) of the block
    const int wg = tid >> 7;
    float acc[KB / 2];
    for (int s = 0; s < NS; ++s) {
      const int slot = s % NST;
      mbar_wait(&ready[slot], (s / NST) & 1);
      const uint32_t sg = smem_u32(smem + slot * stage_bytes) + wg * WT_BOX;  // this warpgroup's 64 gradient channels
      const uint32_t sa = smem_u32(smem + slot * stage_bytes) + a_off;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < WT_BMP / 16; ++kk) {  // 16 pixels = two 8-row swizzle atoms = 2 KB further into every box
        if (KB == 128)
          wgmma_m64n128<1, 1>(acc, desc_mn_sw128(sg + kk * 2048), desc_mn_sw128(sa + kk * 2048), (s > 0 || kk > 0) ? 1u : 0u);
        else
          wgmma_m64n64<1, 1>(acc, desc_mn_sw128(sg + kk * 2048), desc_mn_sw128(sa + kk * 2048), (s > 0 || kk > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous stage's MMAs have read it: it may be refilled
      if (s > 0 && (tid & 127) == 0) mbar_arrive(&empty[(s - 1) % NST]);
    }
    wgmma_wait<0>();
    wgmma_reg_fence<KB / 2>(acc);
    // ---- epilogue: accumulator registers -> fp64 reductions into the dW scratch (fragment: rows 16 w + lane / 4 (+ 8), columns 8 j + 2 (lane % 4))
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = n0 + wg * 64 + ((tid & 127) >> 5) * 16 + (lane >> 2) + 8 * h;
      if (n < p.N) {
        double* __restrict__ dWrow = reinterpret_cast<double*>(p.dW) + (size_t)n * p.lddw;
#pragma unroll
        for (int j = 0; j < KB / 8; ++j) {
          const int k = k0 + 8 * j + 2 * (lane & 3);
          if (k < p.K) atomicAdd(dWrow + k, (double)acc[4 * j + 2 * h]);
          if (k + 1 < p.K) atomicAdd(dWrow + k + 1, (double)acc[4 * j + 2 * h + 1]);
        }
      }
    }
  } else {
    // ===================================================== transform warps
    const int xt = tid - WT_XF0;  // 0..255
    // G role: fixed 16-byte chunk column gc (0..15) of the 128 channels, rows (xt>>4) + 16*i
    const int gc = xt & 15;
    const int gn = n0 + gc * 8;
    const bool gn_ok = gn < p.N;
    const bool want_db = (p.dbias != nullptr) && (blockIdx.y == 0);
    float g0[8], g1[8], g2[8], db[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      g0[e] = (BNB && gn_ok) ? __ldg(p.g_p0 + gn + e) : 1.f;
      g1[e] = (BNB && gn_ok) ? __ldg(p.g_p1 + gn + e) : 0.f;
      g2[e] = (BNB && gn_ok) ? __ldg(p.g_p2 + gn + e) : 0.f;
      db[e] = 0.f;
    }
    // A role: fixed chunk column ac (0..ncc-1), rows (xt / ncc) + rpp*i
    const int ncc = a_boxes * 8;
    const int rpp = 256 / ncc;
    const int ac = xt % ncc, ar0 = xt / ncc;
    const bool a_active = ar0 < rpp;
    const int ak = k0 + ac * 8;
    const bool ak_ok = ak < p.K;
    float ap0[8], ap1[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      ap0[e] = (A_HAS_P && ak_ok) ? __ldg(p.a_p0 + ak + e) : 1.f;
      ap1[e] = (A_HAS_P && ak_ok) ? __ldg(p.a_p1 + ak + e) : 0.f;
    }
    const int rps = p.rows_per_sample > 0 ? p.rows_per_sample : 1;
    const uint32_t g_box = (uint32_t)(gc >> 3) * WT_BOX, a_box = (uint32_t)(ac >> 3) * WT_BOX;

    for (int s = 0; s < NS; ++s) {
      const int slot = s % NST;
      uint8_t* st = smem + slot * stage_bytes;
      mbar_wait(&full[slot], (s / NST) & 1);
      const int mb = m_begin + s * WT_BMP;
      if (BNB || want_db) {
#pragma unroll
        for (int i = 0; i < WT_BMP / 16; ++i) {
          const int row = (xt >> 4) + 16 * i;
          const bool in = mb + row < m_end;
          uint4* pg = reinterpret_cast<uint4*>(st + g_box + sw128(row, gc & 7));
          float f[8];
          unpack8(*pg, f);
          if (BNB) {
            float y[8];
            unpack8(*reinterpret_cast<const uint4*>(st + 2 * WT_BOX + g_box + sw128(row, gc & 7)), y);
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = in ? bf16_round(fmaf(g0[e], f[e], fmaf(g1[e], y[e], g2[e]))) : 0.f;
            *pg = pack8(f);
          }
          if (want_db) {
#pragma unroll
            for (int e = 0; e < 8; ++e) db[e] += in ? f[e] : 0.f;
          }
        }
      }  // RAW gradient: nothing to do (pixel ranges are multiples of the stage, rows past M are zero-filled by TMA)
      if (AMODE != CVB_A_RAW && a_active) {
#pragma unroll 4
        for (int row = ar0; row < WT_BMP; row += rpp) {
          uint4* pa = reinterpret_cast<uint4*>(st + a_off + a_box + sw128(row, ac & 7));
          float f[8];
          unpack8(*pa, f);
          if (AMODE == CVB_A_GN) {
            const int b = min(mb + row, p.M - 1) / rps;
            const float mu = __ldg(p.row_mean + b), rs = __ldg(p.row_rstd + b);
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = fmaf((f[e] - mu) * rs, ap0[e], ap1[e]);
          } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = apply_mode(AMODE, f[e], ap0[e], ap1[e]);
          }
          *pa = pack8(f);  // G' of the rows past m_end is zero, so whatever this produces there cannot reach dW
        }
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
      __syncwarp();
      if (lane == 0) mbar_arrive(&ready[slot]);
    }

    // ---- bias gradient: reduce the thread-local column sums (16 row-threads share a chunk column)
    if (want_db) {
#pragma unroll
      for (int e = 0; e < 8; ++e) atomicAdd(&s_db[gc * 8 + e], (double)db[e]);
      asm volatile("bar.sync 1, %0;" ::"n"(WT_XF_WARPS * 32) : "memory");
      if (xt < 128 && n0 + xt < p.N) atomicAdd(reinterpret_cast<double*>(p.dbias) + n0 + xt, s_db[xt]);
    }

  }
}

template <int GMODE, int AMODE, int KB>
int launch_wgrad_tc(const cvb_wgrad_args& a, cudaStream_t st) {
  // all K blocks of one launch use the same width KB; the last one may be narrower and is padded with zero-filled boxes
  // (K is a multiple of 64 here)
  const int nb = (a.N + 127) / 128, kb = (a.K + WT_KB - 1) / WT_KB;
  const int stage_bytes = ((GMODE == CVB_A_BNB ? 4 : 2) + KB / 64) * WT_BOX;
  int nst = (200 * 1024) / stage_bytes;
  if (nst > WT_MAX_STAGES) nst = WT_MAX_STAGES;
  const int sms = cvb_num_sms();
  int splits = sms / (nb * kb);
  if (splits < 1) splits = 1;
  int max_splits = (a.M + 4 * WT_BMP - 1) / (4 * WT_BMP);  // at least 4 stages per CTA
  if (splits > max_splits) splits = max_splits;
  int m_per_cta = ((a.M + splits - 1) / splits + WT_BMP - 1) / WT_BMP * WT_BMP;
  splits = (a.M + m_per_cta - 1) / m_per_cta;
  const size_t smem = (size_t)nst * stage_bytes + 1024;
  CUtensorMap tmG, tmG2, tmA;
  if (cvb_make_tmap_2d(&tmG, a.G, a.M, a.N, a.ldg, WT_BMP, 64)) return 1;
  if (cvb_make_tmap_2d(&tmG2, GMODE == CVB_A_BNB ? a.G2 : a.G, a.M, a.N, GMODE == CVB_A_BNB ? a.ldg2 : a.ldg, WT_BMP, 64)) return 1;
  if (cvb_make_tmap_2d(&tmA, a.A, a.M, a.K, a.lda, WT_BMP, 64)) return 1;
  CVB_CUDA(cvb_smem_optin<pw_wgrad_tc_kernel<GMODE, AMODE, KB>>(216 * 1024));
  dim3 grid(nb, kb, splits);
  CVB_CUDA(cvb_launch(pw_wgrad_tc_kernel<GMODE, AMODE, KB>, grid, WT_THREADS, smem, st, tmG, tmG2, tmA, a, m_per_cta, nst, stage_bytes));
  return 0;
}

template <int GMODE, int AMODE>
int launch_wgrad_tc(const cvb_wgrad_args& a, cudaStream_t st) {
  return a.K >= WT_KB ? launch_wgrad_tc<GMODE, AMODE, WT_KB>(a, st) : launch_wgrad_tc<GMODE, AMODE, 64>(a, st);
}

template <int GMODE>
int dispatch_wgrad_tc_a(const cvb_wgrad_args& a, cudaStream_t st) {
  switch (a.a_mode) {
    case CVB_A_RAW: return launch_wgrad_tc<GMODE, CVB_A_RAW>(a, st);
    case CVB_A_AFF: return launch_wgrad_tc<GMODE, CVB_A_AFF>(a, st);
    case CVB_A_AFF_SILU: return launch_wgrad_tc<GMODE, CVB_A_AFF_SILU>(a, st);
    case CVB_A_SILU: return launch_wgrad_tc<GMODE, CVB_A_SILU>(a, st);
    case CVB_A_GN: return launch_wgrad_tc<GMODE, CVB_A_GN>(a, st);
    default: return -1;
  }
}

}  // namespace

// Returns 0 when the launch was issued, -1 when the shape is left to the mma.sync kernel, > 0 on error.
int cvb_pw_wgrad_tc(const cvb_wgrad_args& a, cudaStream_t st) {
  // 64-channel TMA boxes on the reduced-over operand: K must be a multiple of 64 (the 3x3 stem / K = 32 layers stay on mma.sync);
  if (a.K % 64 != 0 || a.K < 64 || a.N < 32) return -1;
  if (a.N <= 64 && a.K <= 64) return -1;  // half-empty 128-row block and one 64-column box: left to the 64x64-tile mma.sync kernel
  if (a.g_mode == CVB_A_RAW) return dispatch_wgrad_tc_a<CVB_A_RAW>(a, st);
  if (a.g_mode == CVB_A_BNB) return dispatch_wgrad_tc_a<CVB_A_BNB>(a, st);
  return -1;
}
