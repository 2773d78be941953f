// Pointwise-conv / linear GEMMs for the MobileViTv2 hot path (sm_90a).
//
//   cvb_pw_gemm : C[M,N] = epi( load(A)[M,K] * W[N,K]^T + bias )      forward and input-gradient GEMMs
//   cvb_pw_wgrad: dW[N,K] += sum_m load(G)[m,n] * load(A)[m,k]        weight-gradient GEMM (reduction over pixels)
//
// Every layer here is HBM-bound (K,N <= 768: <= 170 FLOP/B, H100 ridge ~295 FLOP/B from the data sheet's 989 TFLOP/s / 3.35 TB/s; SURVEY.md 8d), so the design goal is
// "read each activation once, write each activation once": the producer's BatchNorm/SiLU/GroupNorm (or the BN-backward of the
// consumer) is a LOAD MODE of the A operand, and bias / activation / residual / BN statistics / GN statistics / activation
// backward / GroupNorm backward are EPILOGUE modes, so no stand-alone normalisation or activation pass exists inside a module.
// This file holds the mma.sync.m16n8k16 (bf16 -> fp32) kernels: the forward / input-gradient GEMM for narrow layers (N < 96) and
// shapes the wgmma kernels do not take, the 64x64-tile weight-gradient kernel (K % 64 != 0 or tiny N, K), and the C-ABI entry
// points that route to the wgmma kernels in gemm_tc.cu and wgrad_tc.cu first.
#include "common.cuh"

namespace {

constexpr int BM = 128;       // CTA tile rows (pixels)
constexpr int BK = 32;        // K step
constexpr int NTHREADS = 256;

__device__ __forceinline__ uint32_t swz64(int row, int ch) {  // 64-byte rows, 4 x 16B chunks
  return static_cast<uint32_t>(row * 64 + ((ch ^ ((row >> 1) & 3)) << 4));
}

// The kernel is INSTRUCTION-ISSUE / latency bound, not tensor bound: K <= 768 gives few MMAs per output
// element, so the design minimises issued instructions per tile and maximises bytes in flight:
//   * operands arrive by TMA (cp.async.bulk.tensor.2d, 64-byte swizzle == the ldmatrix XOR layout): ONE elected thread feeds a
//     ring of A stages that runs across ALL M tiles of the persistent CTA (mbarrier completion); the weight panel [BN, K] is
//     loaded once and stays resident in shared memory;
//   * the prologue (BN+SiLU / GroupNorm / BN-backward) is applied ONCE per element, in place in shared memory, one k-tile
//     ahead of the MMAs (no redundancy across the N-warps);
//   * the epilogue works on the accumulator fragments directly (bias, activation(-backward), residual, statistics), exchanges
//     only bf16 through a padded staging tile (aux tensor in, result out, in place) and copies out with 16-byte row-contiguous
//     stores.
constexpr int MAX_STAGES = 8;

// compile-time epilogue variants (keeps the SASS compact: the generic runtime-switched epilogue was 130 KB of code and stalled
// on instruction fetch)
enum { EPI_STORE = 0, EPI_STORE_R = 1, EPI_SILU = 2, EPI_SILU_BWD = 3, EPI_GN_BWD = 4 };

template <int WM, int AMODE, int EPI>
__global__ void __launch_bounds__(NTHREADS, 2) pw_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                                                              const __grid_constant__ CUtensorMap tmW, const cvb_gemm_args p, int NST) {
  constexpr int WARPS_M = BM / WM;
  constexpr int WARPS_N = 8 / WARPS_M;
  constexpr int BN = WARPS_N * 32;
  constexpr int MI = WM / 16;
  constexpr bool TWO_A = (AMODE == CVB_A_BNB);
  constexpr int A_STAGE = BM * BK * 2;
  constexpr int B_STAGE = BN * BK * 2;
  constexpr int LDO = BN + 8;        // bf16 staging row stride (+16 B: conflict-free fragment access)
  constexpr int CGS = BN / 8;        // 16-byte column groups per row
  constexpr bool HAS_P = (AMODE == CVB_A_AFF || AMODE == CVB_A_AFF_SILU || AMODE == CVB_A_GN || AMODE == CVB_A_BNB);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wm0 = (warp / WARPS_N) * WM;
  const int wn0 = (warp % WARPS_N) * 32;
  const int n0 = blockIdx.x * BN;
  const int KT = (p.K + BK - 1) / BK;
  const int Kpad = KT * BK;
  const int m_tiles = (p.M + BM - 1) / BM;
  const int my_tiles = (m_tiles - (int)blockIdx.y + (int)gridDim.y - 1) / (int)gridDim.y;
  const int total = my_tiles * KT;  // flattened (tile, k-tile) iterations of this CTA

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // swizzled TMA destinations: align by hand
  uint8_t* sW = smem;                                  // resident weight panel: KT blocks of [BN][32]
  uint8_t* sA = sW + KT * B_STAGE;                     // A ring
  uint8_t* sA2 = sA + NST * A_STAGE;                   // second operand of the BN-backward prologue
  uint8_t* sO = sA + (TWO_A ? 2 : 1) * NST * A_STAGE;  // bf16 [BM][LDO] aux-in / result-out staging
  float* sP = reinterpret_cast<float*>(sO + BM * LDO * 2);
  __shared__ double s_col[2][128];
  __shared__ double s_samp[2][128];  // fp64: cross-thread order must not change the GroupNorm statistics
  __shared__ __align__(8) uint64_t full[MAX_STAGES];
  __shared__ __align__(8) uint64_t wbar;

  if (tid < 128) { s_col[0][tid] = 0.0; s_col[1][tid] = 0.0; s_samp[0][tid] = 0.0; s_samp[1][tid] = 0.0; }
  if (tid == 0) {
    for (int i = 0; i < NST; ++i) mbar_init(&full[i], 1);
    mbar_init(&wbar, 1);
    fence_mbar_init();
  }
  pdl_wait();  // everything below may read what the previous kernel wrote
  pdl_trigger();
  if (HAS_P) {  // per-K prologue parameters -> smem (zero padded so that the K tail transforms to zero)
    for (int k = tid; k < Kpad; k += NTHREADS) {
      bool ok = k < p.K;
      sP[k] = ok ? p.a_p0[k] : 0.f;
      sP[Kpad + k] = ok ? p.a_p1[k] : 0.f;
      if (AMODE == CVB_A_BNB) sP[2 * Kpad + k] = ok ? p.a_p2[k] : 0.f;
    }
  }
  __syncthreads();

  const bool want_col = p.col_sum != nullptr;
  const bool want_samp = p.samp_sum != nullptr;
  const int rps = p.rows_per_sample > 0 ? p.rows_per_sample : 1;
  // at most one auxiliary [M, N] tensor: Y (activation / GroupNorm backward) or the residual R
  constexpr bool has_aux = (EPI == EPI_STORE_R || EPI == EPI_SILU_BWD || EPI == EPI_GN_BWD);
  const bf16* __restrict__ AUX = static_cast<const bf16*>(EPI == EPI_STORE_R ? p.R : p.Y);
  const int ldaux = EPI == EPI_STORE_R ? p.ldr : p.ldy;

  float cs[8], cq[8];  // per-column statistics (columns wn0 + ni*8 + 2t + e), accumulated over all tiles, flushed once
#pragma unroll
  for (int j = 0; j < 8; ++j) { cs[j] = 0.f; cq[j] = 0.f; }

  // one ring for the whole CTA lifetime: iteration `it` = (tile it / KT, k-tile it % KT); called by ONE thread
  auto issue = [&](int it) {
    const int stage = it % NST;
    const int j = it / KT, kt = it - j * KT;
    const int m0i = ((int)blockIdx.y + j * (int)gridDim.y) * BM;
    mbar_expect_tx(&full[stage], (TWO_A ? 2 : 1) * A_STAGE);
    tma_load_2d(sA + stage * A_STAGE, &tmA, &full[stage], kt * BK, m0i);  // rows >= M / cols >= K are zero-filled by the TMA unit
    if (TWO_A) tma_load_2d(sA2 + stage * A_STAGE, &tmA2, &full[stage], kt * BK, m0i);
  };
  auto issue_aux = [&](int jt) {  // aux tile of tile jt -> staging buffer (16-byte, row-contiguous)
    const int m0i = ((int)blockIdx.y + jt * (int)gridDim.y) * BM;
    for (int c = tid; c < BM * CGS; c += NTHREADS) {
      int row = c / CGS, cgc = c % CGS;
      int m = m0i + row, n = n0 + cgc * 8;
      bool ok = (m < p.M) && (n < p.N);
      cp_async16(smem_u32(sO + row * (LDO * 2) + cgc * 16), AUX + (ok ? (size_t)m * ldaux + n : 0), ok);
    }
  };
  // in-place prologue of the chunks THIS thread loaded (rows tid>>2 and 64 + tid>>2), one k-tile ahead of the MMAs
  float tmu[2] = {0.f, 0.f}, trs[2] = {1.f, 1.f};
  auto transform = [&](int it) {
    if (AMODE == CVB_A_RAW) return;
    const int stage = it % NST;
    const int j = it / KT, kt = it - j * KT;
    const int k0 = kt * BK;
    const int m0i = ((int)blockIdx.y + j * (int)gridDim.y) * BM;
    if (AMODE == CVB_A_GN && kt == 0) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        int m = m0i + (tid >> 2) + i * 64;
        int b = (m < p.M ? m : p.M - 1) / p.rows_per_sample;
        tmu[i] = __ldg(p.row_mean + b);
        trs[i] = __ldg(p.row_rstd + b);
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int c = tid + i * NTHREADS;
      const int row = c >> 2, ch = c & 3;
      const int k = k0 + ch * 8;
      uint4* pa = reinterpret_cast<uint4*>(sA + stage * A_STAGE + swz64(row, ch));
      float f[8];
      unpack8(*pa, f);
      float q0[8], q1[8];
      if (HAS_P) {
        *reinterpret_cast<float4*>(q0) = *reinterpret_cast<const float4*>(sP + k);
        *reinterpret_cast<float4*>(q0 + 4) = *reinterpret_cast<const float4*>(sP + k + 4);
        *reinterpret_cast<float4*>(q1) = *reinterpret_cast<const float4*>(sP + Kpad + k);
        *reinterpret_cast<float4*>(q1 + 4) = *reinterpret_cast<const float4*>(sP + Kpad + k + 4);
      }
      if (AMODE == CVB_A_AFF) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaf(q0[e], f[e], q1[e]);
      } else if (AMODE == CVB_A_AFF_SILU) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = silu_f(fmaf(q0[e], f[e], q1[e]));
      } else if (AMODE == CVB_A_SILU) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = silu_f(f[e]);
      } else if (AMODE == CVB_A_GN) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaf((f[e] - tmu[i]) * trs[i], q0[e], q1[e]);
      } else {  // BNB: c1*dz + c2*y + c3
        float y[8], q2[8];
        unpack8(*reinterpret_cast<const uint4*>(sA2 + stage * A_STAGE + swz64(row, ch)), y);
        *reinterpret_cast<float4*>(q2) = *reinterpret_cast<const float4*>(sP + 2 * Kpad + k);
        *reinterpret_cast<float4*>(q2 + 4) = *reinterpret_cast<const float4*>(sP + 2 * Kpad + k + 4);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaf(q0[e], f[e], fmaf(q1[e], y[e], q2[e]));
      }
      // rows beyond M must stay exactly zero (their accumulators feed the statistics unmasked)
      *pa = (m0i + row < p.M) ? pack8(f) : make_uint4(0u, 0u, 0u, 0u);
    }
  };

  // ---- prologue of the pipeline
  if (tid == 0) {
    mbar_expect_tx(&wbar, (uint32_t)KT * B_STAGE);
    for (int kt = 0; kt < KT; ++kt) tma_load_2d(sW + kt * B_STAGE, &tmW, &wbar, kt * BK, n0);
    for (int s = 0; s < NST - 1 && s < total; ++s) issue(s);
  }
  if (has_aux && my_tiles > 0) {
    issue_aux(0);
    cp_async_commit();
  }
  mbar_wait(&wbar, 0);
  if (AMODE != CVB_A_RAW && total > 0) {
    mbar_wait(&full[0], 0);
    transform(0);
  }

  int it = 0;
  for (int jt = 0; jt < my_tiles; ++jt) {
    const int m0 = ((int)blockIdx.y + jt * (int)gridDim.y) * BM;
    float acc[MI][4][4];
#pragma unroll
    for (int mi = 0; mi < MI; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0.f;

    for (int kt = 0; kt < KT; ++kt, ++it) {
      if (AMODE != CVB_A_RAW) {
        if (it + 1 < total) mbar_wait(&full[(it + 1) % NST], ((it + 1) / NST) & 1);  // stage it+1 landed (transformed below)
      } else {
        mbar_wait(&full[it % NST], (it / NST) & 1);
      }
      fence_proxy_async();  // order this thread's generic smem accesses before the TMA write that refills a slot
      __syncthreads();      // transform(it) visible; MMAs of it-1 done -> its slot is free
      if (tid == 0) {
        const int nxt = it + NST - 1;
        if (nxt < total) issue(nxt);
      }
      if (AMODE != CVB_A_RAW && it + 1 < total) transform(it + 1);
      const int stage = it % NST;
      const uint32_t aBase = smem_u32(sA + stage * A_STAGE);
      const uint32_t bBase = smem_u32(sW + kt * B_STAGE);
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        uint32_t af[MI][4];
#pragma unroll
        for (int mi = 0; mi < MI; ++mi) {
          int row = wm0 + mi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
          int ch = ks * 2 + (lane >> 4);
          ldmatrix_x4(aBase + swz64(row, ch), af[mi][0], af[mi][1], af[mi][2], af[mi][3]);
        }
        uint32_t bfr[4][2];
#pragma unroll
        for (int nj = 0; nj < 2; ++nj) {
          int row = wn0 + nj * 16 + (lane & 7) + (lane >> 4) * 8;
          int ch = ks * 2 + ((lane >> 3) & 1);
          ldmatrix_x4(bBase + swz64(row, ch), bfr[nj * 2][0], bfr[nj * 2][1], bfr[nj * 2 + 1][0], bfr[nj * 2 + 1][1]);
        }
#pragma unroll
        for (int mi = 0; mi < MI; ++mi)
#pragma unroll
          for (int ni = 0; ni < 4; ++ni) mma_bf16_16816(acc[mi][ni], af[mi], bfr[ni][0], bfr[ni][1]);
      }
    }

    // ------------------------------------------------------------------ epilogue on the accumulator fragments
    if (has_aux) {
      cp_async_wait<0>();  // the aux tile of this tile (issued after the previous copy-out) has landed
      __syncthreads();
    }
    const int first_sample = m0 / rps;
    // per-column vectors of this thread's 8 columns.  Out-of-range columns have zero weights and get zero bias; out-of-range
    // rows have zero A rows and get their bias masked -> every such value is exactly 0 and needs no predicate in the statistics.
    float bias2[4][2], ep0[4][2], ep1[4][2];
#pragma unroll
    for (int ni = 0; ni < 4; ++ni) {
      const int n = n0 + wn0 + ni * 8 + 2 * t;
      const bool nok = n < p.N;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        bias2[ni][e] = (nok && p.bias) ? __ldg(p.bias + n + e) : 0.f;
        if (EPI == EPI_SILU_BWD || EPI == EPI_GN_BWD) ep0[ni][e] = (nok && p.e_p0) ? __ldg(p.e_p0 + n + e) : 1.f;
        if (EPI == EPI_SILU_BWD) ep1[ni][e] = (nok && p.e_p1) ? __ldg(p.e_p1 + n + e) : 0.f;
      }
    }
#pragma unroll
    for (int mi = 0; mi < MI; ++mi)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = wm0 + mi * 16 + g + h * 8;
        const int m = m0 + row;
        const float rmask = m < p.M ? 1.f : 0.f;
        float mu = 0.f, rs = 1.f;
        if (EPI == EPI_GN_BWD) {
          const int b = (m < p.M ? m : p.M - 1) / rps;
          mu = __ldg(p.row_mean + b);
          rs = __ldg(p.row_rstd + b);
        }
        float ssum = 0.f, ssq = 0.f;
        uint32_t* prow = reinterpret_cast<uint32_t*>(sO + row * (LDO * 2) + (wn0 + 2 * t) * 2);
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          float v0 = fmaf(bias2[ni][0], rmask, acc[mi][ni][2 * h]), v1 = fmaf(bias2[ni][1], rmask, acc[mi][ni][2 * h + 1]);
          float y0 = 0.f, y1 = 0.f;
          if (has_aux) { const float2 a2 = unpack_bf162(prow[ni * 4]); y0 = a2.x; y1 = a2.y; }
          if (EPI == EPI_STORE_R) {
            v0 += y0; v1 += y1;
          } else if (EPI == EPI_SILU) {
            v0 = silu_f(v0); v1 = silu_f(v1);
          } else if (EPI == EPI_SILU_BWD) {
            if (p.e_mode != CVB_E_LIN_BWD) {  // LIN_BWD: same statistics, no activation factor (BatchNorm without an activation)
              v0 *= silu_grad_f(fmaf(ep0[ni][0], y0, ep1[ni][0]));
              v1 *= silu_grad_f(fmaf(ep0[ni][1], y1, ep1[ni][1]));
            }
          } else if (EPI == EPI_GN_BWD) {
            y0 = (y0 - mu) * rs; y1 = (y1 - mu) * rs;  // x-hat
            cs[ni * 2] += v0; cs[ni * 2 + 1] += v1;
            cq[ni * 2] = fmaf(v0, y0, cq[ni * 2]); cq[ni * 2 + 1] = fmaf(v1, y1, cq[ni * 2 + 1]);
            v0 *= ep0[ni][0]; v1 *= ep0[ni][1];
          }
          const uint32_t pk = pack_bf162(v0, v1);
          prow[ni * 4] = pk;
          const float2 r = unpack_bf162(pk);  // statistics of the STORED (bf16) values
          if (EPI == EPI_STORE || EPI == EPI_STORE_R || EPI == EPI_SILU) {
            cs[ni * 2] += r.x; cs[ni * 2 + 1] += r.y;
            cq[ni * 2] = fmaf(r.x, r.x, cq[ni * 2]); cq[ni * 2 + 1] = fmaf(r.y, r.y, cq[ni * 2 + 1]);
          } else if (EPI == EPI_SILU_BWD) {
            cs[ni * 2] += r.x; cs[ni * 2 + 1] += r.y;
            cq[ni * 2] = fmaf(r.x, y0, cq[ni * 2]); cq[ni * 2 + 1] = fmaf(r.y, y1, cq[ni * 2 + 1]);
          } else {
            ssum += r.x + r.y;
            ssq = fmaf(r.x, y0, fmaf(r.y, y1, ssq));
          }
        }
        if (EPI == EPI_GN_BWD) {  // per-sample sums of g and g*xhat (GroupNorm backward, phase 1)
          ssum += __shfl_xor_sync(0xffffffffu, ssum, 1); ssum += __shfl_xor_sync(0xffffffffu, ssum, 2);
          ssq += __shfl_xor_sync(0xffffffffu, ssq, 1); ssq += __shfl_xor_sync(0xffffffffu, ssq, 2);
          if (t == 0 && m < p.M && want_samp) {
            const int bi = m / rps - first_sample;
            atomicAdd(&s_samp[0][bi], (double)ssum);
            atomicAdd(&s_samp[1][bi], (double)ssq);
          }
        }
      }
    __syncthreads();  // staged result complete
    {
      bf16* __restrict__ Cg = static_cast<bf16*>(p.C);
      const bool samp_here = want_samp && EPI != EPI_GN_BWD;  // GroupNorm statistics of the stored output, per row of 16-byte chunks
      for (int c = tid; c < BM * CGS; c += NTHREADS) {
        const int row = c / CGS, cgc = c % CGS;
        const int m = m0 + row, n = n0 + cgc * 8;
        const uint4 u = *reinterpret_cast<const uint4*>(sO + row * (LDO * 2) + cgc * 16);
        if (m < p.M && n < p.N) stg16(Cg + (size_t)m * p.ldc + n, u);
        if (samp_here) {
          float f[8];
          unpack8(u, f);
          float sv = 0.f, sq = 0.f;
#pragma unroll
          for (int e = 0; e < 8; ++e) { sv += f[e]; sq = fmaf(f[e], f[e], sq); }
#pragma unroll
          for (int o = CGS / 2; o > 0; o >>= 1) {
            sv += __shfl_xor_sync(0xffffffffu, sv, o);
            sq += __shfl_xor_sync(0xffffffffu, sq, o);
          }
          if (cgc == 0 && m < p.M) {
            const int bi = m / rps - first_sample;
            atomicAdd(&s_samp[0][bi], (double)sv);
            atomicAdd(&s_samp[1][bi], (double)sq);
          }
        }
      }
    }
    if (want_samp) {
      __syncthreads();  // s_samp complete
      if (tid < 128) {
        int mlast = min(m0 + BM, p.M) - 1;
        int nsamp = mlast / rps - first_sample + 1;
        if (tid < nsamp) {
          atomicAdd(p.samp_sum + first_sample + tid, s_samp[0][tid]);
          atomicAdd(p.samp_sq + first_sample + tid, s_samp[1][tid]);
          s_samp[0][tid] = 0.0;
          s_samp[1][tid] = 0.0;
        }
      }
    }
    if (has_aux) {
      __syncthreads();  // copy-out finished: the staging tile may be overwritten by the next tile's aux operand
      if (jt + 1 < my_tiles) { issue_aux(jt + 1); cp_async_commit(); }
    }
    // (without aux the next write to sO happens after >= 1 __syncthreads of the next tile's k-loop)
  }  // tile loop
  cp_async_wait<0>();

  if (want_col) {
    // reduce over the 8 row-lanes (g) that share the columns, then one smem atomic per warp and column
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a = cs[j], q = cq[j];
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        q += __shfl_xor_sync(0xffffffffu, q, o);
      }
      if (g == 0) {
        const int col = wn0 + (j >> 1) * 8 + 2 * t + (j & 1);
        atomicAdd(&s_col[0][col], (double)a);
        atomicAdd(&s_col[1][col], (double)q);
      }
    }
    __syncthreads();
    if (tid < BN && n0 + tid < p.N) {
      atomicAdd(p.col_sum + n0 + tid, s_col[0][tid]);
      atomicAdd(p.col_sq + n0 + tid, s_col[1][tid]);
    }
  }
}

template <int WM, int AMODE, int EPI>
int launch_gemm(const cvb_gemm_args& a, cudaStream_t st, bool require_two_ctas) {
  constexpr int WARPS_M = BM / WM;
  constexpr int BN = (8 / WARPS_M) * 32;
  constexpr int A_STAGE_ALL = BM * BK * 2 * (AMODE == CVB_A_BNB ? 2 : 1);
  const int KT = (a.K + BK - 1) / BK;
  const int nvec = (AMODE == CVB_A_AFF || AMODE == CVB_A_AFF_SILU || AMODE == CVB_A_GN) ? 2 : (AMODE == CVB_A_BNB ? 3 : 0);
  const size_t fixed = (size_t)KT * BN * BK * 2 + (size_t)BM * (BN + 8) * 2 + (size_t)nvec * KT * BK * 4 + 1024;
  // stage count from the shared-memory budget: two CTAs per SM when >= 4 stages fit in half an SM, else one CTA with a deep ring
  int nst = (fixed < (size_t)108 * 1024) ? (int)(((size_t)108 * 1024 - fixed) / A_STAGE_ALL) : 0;
  if (nst < 4) {
    // one CTA per SM serialises main loop and epilogue (measured 3-4x slower per tile): let the caller try a narrower N tile first
    if (require_two_ctas) return -1;
    nst = (fixed < (size_t)216 * 1024) ? (int)(((size_t)216 * 1024 - fixed) / A_STAGE_ALL) : 0;
  }
  if (nst > MAX_STAGES) nst = MAX_STAGES;
  // the transform-ahead pipeline waits for stage it+1 before issuing stage it+NST-1: it needs >= 3 stages
  if (nst < 3) return -1;  // caller retries with a narrower N tile (smaller resident weight panel)
  size_t smem = fixed + (size_t)nst * A_STAGE_ALL;
  static bool attr_set = false;
  if (!attr_set) {
    CVB_CUDA(cudaFuncSetAttribute(pw_gemm_kernel<WM, AMODE, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));
    attr_set = true;
  }
  // resident CTAs per SM: registers allow 2 (launch bounds); shared memory: 228 KB per SM, ~5 KB static + reserved per CTA
  const int occ = (2 * (smem + 5 * 1024) <= (size_t)228 * 1024) ? 2 : 1;
  const int n_tiles = (a.N + BN - 1) / BN, m_tiles = (a.M + BM - 1) / BM;
  int gy = (occ * cvb_num_sms()) / n_tiles;  // all CTAs resident (never more than fit at once), each streaming over its M tiles
  if (gy > m_tiles) gy = m_tiles;
  if (gy < 1) gy = 1;
  CUtensorMap tmA, tmA2, tmW;
  if (cvb_make_tmap_2d_k32(&tmA, a.A, a.M, a.K, a.lda, BM)) return 1;
  if (cvb_make_tmap_2d_k32(&tmA2, AMODE == CVB_A_BNB ? a.A2 : a.A, a.M, a.K, AMODE == CVB_A_BNB ? a.lda2 : a.lda, BM)) return 1;
  if (cvb_make_tmap_2d_k32(&tmW, a.W, a.N, a.K, a.ldw, BN)) return 1;
  dim3 grid(n_tiles, gy);
  CVB_CUDA(cvb_launch(pw_gemm_kernel<WM, AMODE, EPI>, grid, NTHREADS, smem, st, tmA, tmA2, tmW, a, nst));
  CVB_LAUNCH_CHECK();
  return 0;
}

template <int AMODE, int EPI>
int dispatch_tile(const cvb_gemm_args& a, cudaStream_t st) {
  const int N = a.N;
  const int pad128 = (N + 127) / 128 * 128, pad64 = (N + 63) / 64 * 64;
  const bool want128 = N > 64 && pad64 >= pad128;
  int rc = -1;
  // first choice: the widest N tile that still leaves room for two resident CTAs per SM with a >= 4-stage ring
  if (want128) rc = launch_gemm<64, AMODE, EPI>(a, st, true);              // BN = 128
  if (rc == -1 && N > 32) rc = launch_gemm<32, AMODE, EPI>(a, st, true);   // BN = 64
  if (rc == -1 && N <= 32) rc = launch_gemm<16, AMODE, EPI>(a, st, true);  // BN = 32
  // otherwise one CTA per SM with a deep ring
  if (rc == -1 && want128) rc = launch_gemm<64, AMODE, EPI>(a, st, false);
  if (rc == -1 && N > 32) rc = launch_gemm<32, AMODE, EPI>(a, st, false);
  if (rc == -1) rc = launch_gemm<16, AMODE, EPI>(a, st, false);
  return rc;  // -1: K is too large for the resident weight panel of every N tile
}

// the (prologue, epilogue) combinations the hot path uses (functional.py) plus STORE / STORE_R for every prologue
template <int AMODE>
int dispatch_epi(const cvb_gemm_args& a, int epi, cudaStream_t st) {
  if (epi == EPI_STORE) return dispatch_tile<AMODE, EPI_STORE>(a, st);
  if (epi == EPI_STORE_R) return dispatch_tile<AMODE, EPI_STORE_R>(a, st);
  if (AMODE == CVB_A_RAW || AMODE == CVB_A_BNB) {
    if (epi == EPI_SILU_BWD) return dispatch_tile<AMODE, EPI_SILU_BWD>(a, st);
    if (epi == EPI_GN_BWD) return dispatch_tile<AMODE, EPI_GN_BWD>(a, st);
  }
  if (AMODE == CVB_A_RAW && epi == EPI_SILU) return dispatch_tile<CVB_A_RAW, EPI_SILU>(a, st);
  cvb_set_error("cvb_pw_gemm: load mode %d with epilogue %d is not instantiated", AMODE, epi);
  return 1;
}

// =====================================================================================================================
// weight gradient
// =====================================================================================================================
constexpr int WG_TN = 64, WG_TK = 64, WG_MB = 64, WG_STAGES = 4;

__device__ __forceinline__ uint32_t swz128(int row, int ch) {  // 128-byte rows, 8 x 16B chunks
  return static_cast<uint32_t>(row * 128 + ((ch ^ (row & 7)) << 4));
}

template <int GMODE, int AMODE>
__global__ void __launch_bounds__(NTHREADS, 2) pw_wgrad_kernel(const cvb_wgrad_args p, int m_per_cta) {
  constexpr bool TWO_G = (GMODE == CVB_A_BNB);
  constexpr bool A_HAS_P = (AMODE == CVB_A_AFF || AMODE == CVB_A_AFF_SILU || AMODE == CVB_A_GN);
  constexpr int T_STAGE = WG_MB * 64 * 2;  // bytes per operand tile and stage
  constexpr int NST = WG_STAGES;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sG = smem;
  uint8_t* sG2 = smem + NST * T_STAGE;
  uint8_t* sA = smem + (TWO_G ? 2 : 1) * NST * T_STAGE;
  __shared__ double s_db[WG_TN];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wn0 = (warp >> 2) * 32;  // 2 warps along n
  const int wk0 = (warp & 3) * 16;   // 4 warps along k
  const int k0 = blockIdx.x * WG_TK;
  const int n0 = blockIdx.y * WG_TN;
  const int m_begin = blockIdx.z * m_per_cta;
  const int m_end = min(p.M, m_begin + m_per_cta);
  const int NS = (m_end - m_begin + WG_MB - 1) / WG_MB;
  pdl_wait();
  pdl_trigger();
  if (NS <= 0) return;

  const bf16* __restrict__ G = static_cast<const bf16*>(p.G);
  const bf16* __restrict__ G2 = static_cast<const bf16*>(p.G2);
  const bf16* __restrict__ A = static_cast<const bf16*>(p.A);
  const bool want_db = (p.dbias != nullptr) && (blockIdx.x == 0);
  if (tid < WG_TN) s_db[tid] = 0.0;

  // loader / transformer role: this thread owns chunk column `lch` (8 channels) of rows (tid>>3) + 32*i of every stage
  const int lch = tid & 7;
  const int ln = n0 + lch * 8, lk = k0 + lch * 8;
  const bool ln_ok = ln < p.N, lk_ok = lk < p.K;
  float gp0[8], gp1[8], gp2[8], ap0[8], ap1[8], db[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    gp0[e] = (TWO_G && ln_ok) ? __ldg(p.g_p0 + ln + e) : 1.f;
    gp1[e] = (TWO_G && ln_ok) ? __ldg(p.g_p1 + ln + e) : 0.f;
    gp2[e] = (TWO_G && ln_ok) ? __ldg(p.g_p2 + ln + e) : 0.f;
    ap0[e] = (A_HAS_P && lk_ok) ? __ldg(p.a_p0 + lk + e) : 1.f;
    ap1[e] = (A_HAS_P && lk_ok) ? __ldg(p.a_p1 + lk + e) : 0.f;
    db[e] = 0.f;
  }
  const int rps = p.rows_per_sample > 0 ? p.rows_per_sample : 1;

  auto load_stage = [&](int s) {
    const int stage = s % NST;
#pragma unroll
    for (int i = 0; i < WG_MB / 32; ++i) {
      const int row = (tid >> 3) + i * 32;
      const int m = m_begin + s * WG_MB + row;
      const bool okg = (m < m_end) && ln_ok, oka = (m < m_end) && lk_ok;
      cp_async16(smem_u32(sG + stage * T_STAGE) + swz128(row, lch), G + (okg ? (size_t)m * p.ldg + ln : 0), okg);
      if (TWO_G) cp_async16(smem_u32(sG2 + stage * T_STAGE) + swz128(row, lch), G2 + (okg ? (size_t)m * p.ldg2 + ln : 0), okg);
      cp_async16(smem_u32(sA + stage * T_STAGE) + swz128(row, lch), A + (oka ? (size_t)m * p.lda + lk : 0), oka);
    }
  };
  // in-place operand transforms of this thread's own chunks (once per element; the MMA warps then only ldmatrix + mma)
  auto transform = [&](int s) {
    const int stage = s % NST;
#pragma unroll
    for (int i = 0; i < WG_MB / 32; ++i) {
      const int row = (tid >> 3) + i * 32;
      const int m = m_begin + s * WG_MB + row;
      const bool in = m < m_end;
      if (TWO_G || want_db) {
        uint4* pg = reinterpret_cast<uint4*>(sG + stage * T_STAGE + swz128(row, lch));
        float f[8];
        unpack8(*pg, f);
        if (TWO_G) {
          float y[8];
          unpack8(*reinterpret_cast<const uint4*>(sG2 + stage * T_STAGE + swz128(row, lch)), y);
#pragma unroll
          for (int e = 0; e < 8; ++e) f[e] = in ? bf16_round(fmaf(gp0[e], f[e], fmaf(gp1[e], y[e], gp2[e]))) : 0.f;
          *pg = pack8(f);
        }
        if (want_db) {
#pragma unroll
          for (int e = 0; e < 8; ++e) db[e] += f[e];  // rows beyond m_end are zero (zero fill / masked above)
        }
      }
      if (AMODE != CVB_A_RAW) {
        uint4* pa = reinterpret_cast<uint4*>(sA + stage * T_STAGE + swz128(row, lch));
        float f[8];
        unpack8(*pa, f);
        if (AMODE == CVB_A_GN) {
          const int b = min(m, p.M - 1) / rps;
          const float mu = __ldg(p.row_mean + b), rs = __ldg(p.row_rstd + b);
#pragma unroll
          for (int e = 0; e < 8; ++e) f[e] = fmaf((f[e] - mu) * rs, ap0[e], ap1[e]);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) f[e] = apply_mode(AMODE, f[e], ap0[e], ap1[e]);
        }
        *pa = pack8(f);  // G' of the tail rows is zero, so garbage here cannot reach dW
      }
    }
  };

  float acc[2][2][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[a][b][e] = 0.f;

#pragma unroll
  for (int s = 0; s < NST - 1; ++s) {
    if (s < NS) load_stage(s);
    cp_async_commit();
  }
  cp_async_wait<NST - 2>();
  transform(0);
  for (int s = 0; s < NS; ++s) {
    cp_async_wait<NST - 3>();  // own chunks of stage s+1 landed
    __syncthreads();           // transform(s) visible; MMAs of s-1 done
    {
      int ns = s + NST - 1;
      if (ns < NS) load_stage(ns);
      cp_async_commit();
    }
    if (s + 1 < NS) transform(s + 1);
    const int stage = s % NST;
    const uint32_t gBase = smem_u32(sG + stage * T_STAGE), aBase = smem_u32(sA + stage * T_STAGE);
#pragma unroll
    for (int ms = 0; ms < WG_MB / 16; ++ms) {
      uint32_t gf[2][4];
#pragma unroll
      for (int ni = 0; ni < 2; ++ni) {
        int row = ms * 16 + (lane & 7) + (lane >> 4) * 8;
        int ch = (wn0 + ni * 16) / 8 + ((lane >> 3) & 1);
        ldmatrix_x4_trans(gBase + swz128(row, ch), gf[ni][0], gf[ni][1], gf[ni][2], gf[ni][3]);
      }
      uint32_t af[4];
      {
        int row = ms * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        int ch = wk0 / 8 + (lane >> 4);
        ldmatrix_x4_trans(aBase + swz128(row, ch), af[0], af[1], af[2], af[3]);
      }
#pragma unroll
      for (int ni = 0; ni < 2; ++ni)
#pragma unroll
        for (int kj = 0; kj < 2; ++kj) mma_bf16_16816(acc[ni][kj], gf[ni], af[kj * 2], af[kj * 2 + 1]);
    }
  }
  cp_async_wait<0>();

#pragma unroll
  for (int ni = 0; ni < 2; ++ni)
#pragma unroll
    for (int kj = 0; kj < 2; ++kj)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int n = n0 + wn0 + ni * 16 + g + (e >> 1) * 8;
        int k = k0 + wk0 + kj * 8 + 2 * t + (e & 1);
        if (n < p.N && k < p.K) atomicAdd(reinterpret_cast<double*>(p.dW) + (size_t)n * p.lddw + k, (double)acc[ni][kj][e]);
      }
  if (want_db) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float v = db[e];  // reduce over the 4 row-lanes of this warp that share the chunk column (lane bits 3,4)
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      if (lane < 8) atomicAdd(&s_db[lch * 8 + e], (double)v);
    }
    __syncthreads();
    if (tid < WG_TN && n0 + tid < p.N) atomicAdd(reinterpret_cast<double*>(p.dbias) + n0 + tid, s_db[tid]);
  }
}

template <int GMODE, int AMODE>
int launch_wgrad(const cvb_wgrad_args& a, cudaStream_t st) {
  const int kt = (a.K + WG_TK - 1) / WG_TK, nt = (a.N + WG_TN - 1) / WG_TN;
  const int target = 4 * cvb_num_sms();
  int splits = (target + kt * nt - 1) / (kt * nt);
  int max_splits = (a.M + 255) / 256;  // at least 256 rows per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int m_per_cta = ((a.M + splits - 1) / splits + WG_MB - 1) / WG_MB * WG_MB;
  splits = (a.M + m_per_cta - 1) / m_per_cta;
  size_t smem = (size_t)WG_STAGES * WG_MB * 64 * 2 * (GMODE == CVB_A_BNB ? 3 : 2);
  static bool attr_set = false;
  if (!attr_set) {
    CVB_CUDA(cudaFuncSetAttribute(pw_wgrad_kernel<GMODE, AMODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
    attr_set = true;
  }
  dim3 grid(kt, nt, splits);
  CVB_CUDA(cvb_launch(pw_wgrad_kernel<GMODE, AMODE>, grid, NTHREADS, smem, st, a, m_per_cta));
  CVB_LAUNCH_CHECK();
  return 0;
}

template <int GMODE>
int dispatch_wgrad_a(const cvb_wgrad_args& a, cudaStream_t st) {
  switch (a.a_mode) {
    case CVB_A_RAW: return launch_wgrad<GMODE, CVB_A_RAW>(a, st);
    case CVB_A_AFF: return launch_wgrad<GMODE, CVB_A_AFF>(a, st);
    case CVB_A_AFF_SILU: return launch_wgrad<GMODE, CVB_A_AFF_SILU>(a, st);
    case CVB_A_SILU: return launch_wgrad<GMODE, CVB_A_SILU>(a, st);
    case CVB_A_GN: return launch_wgrad<GMODE, CVB_A_GN>(a, st);
    default: cvb_set_error("cvb_pw_wgrad: unsupported a_mode %d", a.a_mode); return 1;
  }
}

}  // namespace

int cvb_pw_wgrad_tc(const cvb_wgrad_args& a, cudaStream_t st);  // wgrad_tc.cu: wgmma weight-gradient kernel
int cvb_pw_gemm_tc(const cvb_gemm_args& a, cudaStream_t st, bool any_n);  // gemm_tc.cu: wgmma kernel (all load modes; STORE / residual / SiLU-backward / GroupNorm-backward epilogues)
static int g_tc_enabled = 1;
extern "C" int cvb_set_tc_enabled(int on) {
  int old = g_tc_enabled;
  g_tc_enabled = on ? 1 : 0;
  return old;
}

extern "C" int cvb_pw_gemm(const cvb_gemm_args* args, cvb_stream_t stream) {
  CVB_CHECK(args != nullptr, "cvb_pw_gemm: null args");
  const cvb_gemm_args& a = *args;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CVB_CHECK(a.M > 0 && a.N > 0 && a.K > 0, "cvb_pw_gemm: bad shape M=%d N=%d K=%d", a.M, a.N, a.K);
  CVB_CHECK(a.K % 8 == 0 && a.N % 8 == 0, "cvb_pw_gemm: K (%d) and N (%d) must be multiples of 8", a.K, a.N);
  CVB_CHECK(a.lda % 8 == 0 && a.ldw % 8 == 0 && a.ldc % (a.c_fp32 ? 4 : 8) == 0, "cvb_pw_gemm: leading dims must be multiples of 8");
  CVB_CHECK(a.A && a.W && a.C, "cvb_pw_gemm: null operand");
  CVB_CHECK(cvb_aligned16(a.A) && cvb_aligned16(a.W) && cvb_aligned16(a.C), "cvb_pw_gemm: operands must be 16-byte aligned");
  CVB_CHECK(a.e_mode >= CVB_E_STORE && a.e_mode <= CVB_E_LIN_BWD, "cvb_pw_gemm: bad e_mode %d", a.e_mode);
  CVB_CHECK(!a.c_fp32, "cvb_pw_gemm: fp32 output is not supported (activations and logits are bf16 like the reference under autocast)");
  CVB_CHECK(!(a.R && a.e_mode >= CVB_E_SILU_BWD), "cvb_pw_gemm: a residual cannot be combined with the backward epilogues");
  if (a.e_mode == CVB_E_SILU_BWD || a.e_mode == CVB_E_GN_BWD || a.e_mode == CVB_E_LIN_BWD)
    CVB_CHECK(a.Y && a.ldy % 8 == 0 && cvb_aligned16(a.Y), "cvb_pw_gemm: epilogue mode %d needs Y", a.e_mode);
  if (a.e_mode == CVB_E_GN_BWD || a.a_mode == CVB_A_GN)
    CVB_CHECK(a.row_mean && a.row_rstd && a.rows_per_sample > 0, "cvb_pw_gemm: GroupNorm modes need row_mean/row_rstd/rows_per_sample");
  if (a.R) CVB_CHECK(a.ldr % 8 == 0 && cvb_aligned16(a.R), "cvb_pw_gemm: bad residual");
  if (a.samp_sum) CVB_CHECK(a.samp_sq && a.rows_per_sample > 0, "cvb_pw_gemm: sample statistics need rows_per_sample");
  if (a.col_sum) CVB_CHECK(a.col_sq != nullptr, "cvb_pw_gemm: col_sq missing");
  CVB_CHECK(!(a.R && a.e_mode == CVB_E_SILU), "cvb_pw_gemm: SiLU epilogue with a residual is not instantiated");
  if (a.a_mode == CVB_A_AFF || a.a_mode == CVB_A_AFF_SILU || a.a_mode == CVB_A_GN) CVB_CHECK(a.a_p0 && a.a_p1, "cvb_pw_gemm: load mode %d needs p0/p1", a.a_mode);
  if (a.a_mode == CVB_A_BNB)
    CVB_CHECK(a.A2 && a.a_p0 && a.a_p1 && a.a_p2 && a.lda2 % 8 == 0 && cvb_aligned16(a.A2), "cvb_pw_gemm: BNB needs A2 and p0/p1/p2");
  if (g_tc_enabled) {
    int rc = cvb_pw_gemm_tc(a, st, false);  // wgmma kernel: STORE / residual / SiLU-backward epilogues, N >= 96
    if (rc != -1) return rc;
  }
  const int epi = a.e_mode == CVB_E_STORE ? (a.R ? EPI_STORE_R : EPI_STORE) : a.e_mode == CVB_E_SILU ? EPI_SILU
                  : (a.e_mode == CVB_E_SILU_BWD || a.e_mode == CVB_E_LIN_BWD) ? EPI_SILU_BWD : EPI_GN_BWD;
  int rc;
  switch (a.a_mode) {
    case CVB_A_RAW: rc = dispatch_epi<CVB_A_RAW>(a, epi, st); break;
    case CVB_A_AFF: CVB_CHECK(a.a_p0 && a.a_p1, "cvb_pw_gemm: AFF needs p0/p1"); rc = dispatch_epi<CVB_A_AFF>(a, epi, st); break;
    case CVB_A_AFF_SILU: CVB_CHECK(a.a_p0 && a.a_p1, "cvb_pw_gemm: AFF_SILU needs p0/p1"); rc = dispatch_epi<CVB_A_AFF_SILU>(a, epi, st); break;
    case CVB_A_SILU: rc = dispatch_epi<CVB_A_SILU>(a, epi, st); break;
    case CVB_A_GN: CVB_CHECK(a.a_p0 && a.a_p1, "cvb_pw_gemm: GN needs gamma/beta"); rc = dispatch_epi<CVB_A_GN>(a, epi, st); break;
    case CVB_A_BNB:
      CVB_CHECK(a.A2 && a.a_p0 && a.a_p1 && a.a_p2 && a.lda2 % 8 == 0 && cvb_aligned16(a.A2), "cvb_pw_gemm: BNB needs A2 and p0/p1/p2");
      rc = dispatch_epi<CVB_A_BNB>(a, epi, st);
      break;
    default: cvb_set_error("cvb_pw_gemm: unsupported a_mode %d", a.a_mode); return 1;
  }
  // a narrow layer whose K does not fit the mma.sync kernel's resident weight panel (the EfficientNet-b6 / b7 squeeze-excitation reduce
  // convs: K = 3456 / 3840): the wgmma kernel streams the weight k-blocks through its ring
  if (rc == -1 && g_tc_enabled) rc = cvb_pw_gemm_tc(a, st, true);
  CVB_CHECK(rc != -1, "cvb_pw_gemm: K=%d is too large for the resident weight panel", a.K);
  return rc;
}

extern "C" int cvb_pw_wgrad(const cvb_wgrad_args* args, cvb_stream_t stream) {
  CVB_CHECK(args != nullptr, "cvb_pw_wgrad: null args");
  const cvb_wgrad_args& a = *args;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CVB_CHECK(a.M > 0 && a.N > 0 && a.K > 0, "cvb_pw_wgrad: bad shape M=%d N=%d K=%d", a.M, a.N, a.K);
  CVB_CHECK(a.K % 8 == 0 && a.N % 8 == 0, "cvb_pw_wgrad: K (%d) and N (%d) must be multiples of 8", a.K, a.N);
  CVB_CHECK(a.G && a.A && a.dW, "cvb_pw_wgrad: null operand");
  CVB_CHECK(a.ldg % 8 == 0 && a.lda % 8 == 0 && cvb_aligned16(a.G) && cvb_aligned16(a.A), "cvb_pw_wgrad: operands must be 16-byte aligned / ld % 8");
  if (a.a_mode == CVB_A_GN) CVB_CHECK(a.row_mean && a.row_rstd && a.rows_per_sample > 0 && a.a_p0 && a.a_p1, "cvb_pw_wgrad: GN needs statistics");
  if (a.a_mode == CVB_A_AFF || a.a_mode == CVB_A_AFF_SILU) CVB_CHECK(a.a_p0 && a.a_p1, "cvb_pw_wgrad: AFF needs p0/p1");
  if (a.g_mode == CVB_A_BNB) CVB_CHECK(a.G2 && a.g_p0 && a.g_p1 && a.g_p2 && a.ldg2 % 8 == 0 && cvb_aligned16(a.G2), "cvb_pw_wgrad: BNB needs G2 and p0/p1/p2");
  CVB_CHECK(a.g_mode == CVB_A_RAW || a.g_mode == CVB_A_BNB, "cvb_pw_wgrad: unsupported g_mode %d", a.g_mode);
  // the kernels reduce split partials with fp64 atomics into a scratch (order-independent), which is then added to dW / dbias
  double* ws = nullptr;
  const size_t nW = (size_t)a.N * a.K;
  if (cvb_det_alloc(&ws, nW + (a.dbias ? a.N : 0), st)) return 2;
  cvb_wgrad_args b = a;
  b.dW = reinterpret_cast<float*>(ws);
  b.lddw = a.K;
  b.dbias = a.dbias ? reinterpret_cast<float*>(ws + nW) : nullptr;
  int rc = -1;
  if (g_tc_enabled) rc = cvb_pw_wgrad_tc(b, st);  // wgmma kernel: whole [128 x 128] dW blocks in registers, operands read once
  if (rc < 0) rc = a.g_mode == CVB_A_RAW ? dispatch_wgrad_a<CVB_A_RAW>(b, st) : dispatch_wgrad_a<CVB_A_BNB>(b, st);
  if (rc == 0) rc = cvb_det_add(ws, a.dW, a.N, a.K, a.lddw, st);
  if (rc == 0 && a.dbias) rc = cvb_det_add(ws + nW, a.dbias, 1, a.N, a.N, st);
  const int rf = cvb_det_free(ws, st);
  return rc ? rc : rf;
}
