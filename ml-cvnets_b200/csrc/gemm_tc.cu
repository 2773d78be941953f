// wgmma / TMA pointwise-conv GEMM (sm_90a): every load mode, STORE / residual / SiLU-backward / GroupNorm-backward epilogues.
//
//   C[M,N] = epi( A[M,K] * W[N,K]^T + bias )          same contract as the mma.sync kernel in gemm.cu
//
// Warp-specialised, one persistent CTA per SM:
//   warps 0-7  two consumer warpgroups: warpgroup g issues wgmma.m64n128k16 for output channels [64 g, 64 g + 64) of the tile
//              (fp32 accumulator in registers), then runs the epilogue on those registers: bias / residual / activation-backward /
//              BatchNorm statistics, bf16 staging tile in smem, 16-byte row-contiguous stores
//   warp 8     TMA producer : ring of A stages [128 pixels x 32 k] (cp.async.bulk.tensor.2d, 64-byte swizzle) across ALL tiles
//   warps 9-   transform    : (layers with a prologue) apply the producer's BN(+SiLU) / GroupNorm / BN-backward to the landed A
//                             stage in place, fence.proxy.async, then hand the stage to the consumers through a second mbarrier
// The product is computed TRANSPOSED, D[channel, pixel] = W[channel, :] . A[pixel, :], i.e. the weight panel is the wgmma "A"
// operand (M = 64 output channels per warpgroup) and the activation tile the "B" operand (N = 128 pixels).  Each consumer thread
// owns two output channels and 32 pixels of each: bias is a pair of scalars and the per-channel BatchNorm sums stay in registers
// until the CTA's last tile (one quad shuffle, then one fp64 atomic per channel per CTA).  The TMA loads of tiles j+1... overlap
// the epilogue of tile j.
#include "common.cuh"

namespace {

constexpr int TC_BM = 128;      // pixels per tile  (wgmma N)
constexpr int TC_BN = 128;      // channels per tile (2 warpgroups x wgmma M 64)
constexpr int TC_BK = 32;       // k per stage (64-byte rows)
constexpr int TC_STAGE = TC_BM * TC_BK * 2;   // 8 KB
constexpr int TC_WBLK = TC_BN * TC_BK * 2;    // 8 KB per k-block of the weight panel
constexpr int TC_LDO = TC_BN + 8;             // bf16 staging row stride (elements)
constexpr int TC_EPI_THREADS = 256;           // the two consumer warpgroups
constexpr int TC_PRODUCER_WARP = TC_EPI_THREADS / 32;
constexpr int TC_THREADS = TC_EPI_THREADS + 32;
constexpr int TC_XF_THREADS_MAX = 256;      // transform warps (only launched for layers with a prologue).  Each warp is a latency-bound
                                            // chain (LDS -> convert -> FMA -> MUFU -> pack -> STS), so the prologue layers run 8 warps; the
                                            // BNB prologue (two operand tiles per stage, SiLU-backward epilogue) runs 4
template <int AMODE>
struct XfCfg {
  static constexpr int THREADS = (AMODE == CVB_A_RAW) ? 0 : (AMODE == CVB_A_BNB ? 128 : TC_XF_THREADS_MAX);
  static constexpr int IT = THREADS ? (TC_BM * 4) / THREADS : 1;  // 16-byte chunks of a [128 x 32] bf16 stage per transform thread
};
constexpr int TC_MAX_STAGES = 12;

enum { TEPI_STORE = 0, TEPI_STORE_R = 1, TEPI_SILU_BWD = 2, TEPI_GN_BWD = 3 };

// K-major operand, 64-byte swizzle: rows of 64 B (32 k), 8-row groups 512 B apart; a k-step of 16 advances the start by 32 B
__device__ __forceinline__ uint64_t desc_sw64(uint32_t saddr) { return wgmma_desc(saddr, 16, 512, WG_SW64); }
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(TC_EPI_THREADS) : "memory"); }

// WRES: the weight panel [128 ch, K] stays resident in smem (loaded once); otherwise (large K) its k-blocks stream through the
// ring next to the activation k-blocks (they are L2 hits: every CTA of an N tile reads the same panel).
template <int AMODE, int EPI, bool WRES>
__global__ void __launch_bounds__(TC_THREADS + XfCfg<AMODE>::THREADS, 1)
    pw_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmW,
                      const cvb_gemm_args p, int NST) {
  constexpr bool XF = (AMODE != CVB_A_RAW);     // has transform warps
  constexpr bool TWO_A = (AMODE == CVB_A_BNB);  // BN-backward prologue streams two tensors
  constexpr bool HAS_P = (AMODE == CVB_A_AFF || AMODE == CVB_A_AFF_SILU || AMODE == CVB_A_GN || AMODE == CVB_A_BNB);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = blockIdx.x * TC_BN;
  const int KT = (p.K + TC_BK - 1) / TC_BK;
  const int m_tiles = (p.M + TC_BM - 1) / TC_BM;
  const int my_tiles = (m_tiles - (int)blockIdx.y + (int)gridDim.y - 1) / (int)gridDim.y;
  const int total = my_tiles * KT;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int A_BYTES = (TWO_A ? 2 : 1) * TC_STAGE;
  constexpr int RING_STAGE = A_BYTES + (WRES ? 0 : TC_WBLK);  // [A | A2 (BNB) | W block (streaming)]
  uint8_t* sW = smem;                               // resident weight panel: KT blocks [128 ch][32 k] (WRES only)
  uint8_t* sA = sW + (WRES ? KT * TC_WBLK : 0);     // ring
  uint8_t* sO = sA + NST * RING_STAGE;              // bf16 [128 pix][TC_LDO] staging (aux in / result out)
  float* sP = reinterpret_cast<float*>(sO + TC_BM * TC_LDO * 2);  // prologue parameters [3][Kpad]
  __shared__ __align__(8) uint64_t full[TC_MAX_STAGES], empty[TC_MAX_STAGES], ready[TC_MAX_STAGES];
  __shared__ __align__(8) uint64_t wbar;
  __shared__ double s_samp[2][128];

  if (tid == 0) {
    for (int i = 0; i < NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 2); mbar_init(&ready[i], XfCfg<AMODE>::THREADS ? XfCfg<AMODE>::THREADS / 32 : 1); }
    mbar_init(&wbar, 1);
    fence_mbar_init();
  }
  if (tid < 128) { s_samp[0][tid] = 0.0; s_samp[1][tid] = 0.0; }
  __syncthreads();
  pdl_wait();  // barriers and CTA scheduling overlapped the previous kernel's tail; data accesses start here
  pdl_trigger();

  if (warp == TC_PRODUCER_WARP) {
    // ===================================================== TMA producer
    if (lane == 0) {
      if (WRES) {
        mbar_expect_tx(&wbar, (uint32_t)KT * TC_WBLK);
        for (int kt = 0; kt < KT; ++kt) tma_load_2d(sW + kt * TC_WBLK, &tmW, &wbar, kt * TC_BK, n0);
      }
      for (int it = 0; it < total; ++it) {
        const int stage = it % NST;
        if (it >= NST) mbar_wait(&empty[stage], ((it / NST) - 1) & 1);  // MMAs that read this slot have completed
        const int j = it / KT, kt = it - j * KT;
        const int m0 = ((int)blockIdx.y + j * (int)gridDim.y) * TC_BM;
        mbar_expect_tx(&full[stage], RING_STAGE);
        tma_load_2d(sA + stage * RING_STAGE, &tmA, &full[stage], kt * TC_BK, m0);
        if (TWO_A) tma_load_2d(sA + stage * RING_STAGE + TC_STAGE, &tmA2, &full[stage], kt * TC_BK, m0);
        if (!WRES) tma_load_2d(sA + stage * RING_STAGE + A_BYTES, &tmW, &full[stage], kt * TC_BK, n0);
      }
    }
  } else if (warp > TC_PRODUCER_WARP) {
    // ===================================================== transform warps: producer's normalisation / activation, in place
    if (XF) {
      constexpr int TC_XF_THREADS = XfCfg<AMODE>::THREADS > 0 ? XfCfg<AMODE>::THREADS : 128;
      constexpr int TC_XF_IT = XfCfg<AMODE>::IT;
      const int tt = tid - TC_THREADS;  // 0..TC_XF_THREADS-1
      const int Kpad = KT * TC_BK;
      if (HAS_P) {
        for (int k = tt; k < Kpad; k += TC_XF_THREADS) {
          const bool ok = k < p.K;
          sP[k] = ok ? p.a_p0[k] : 0.f;
          sP[Kpad + k] = ok ? p.a_p1[k] : 0.f;
          if (AMODE == CVB_A_BNB) sP[2 * Kpad + k] = ok ? p.a_p2[k] : 0.f;
        }
        asm volatile("bar.sync 2, %0;" ::"n"(TC_XF_THREADS) : "memory");
      }
      float tmu[TC_XF_IT], trs[TC_XF_IT];
#pragma unroll
      for (int i = 0; i < TC_XF_IT; ++i) { tmu[i] = 0.f; trs[i] = 1.f; }
      for (int it = 0; it < total; ++it) {
        const int stage = it % NST;
        const int j = it / KT, kt = it - j * KT;
        const int m0 = ((int)blockIdx.y + j * (int)gridDim.y) * TC_BM;
        const int k0 = kt * TC_BK;
        if (AMODE == CVB_A_GN && kt == 0) {
#pragma unroll
          for (int i = 0; i < TC_XF_IT; ++i) {
            const int m = m0 + (tt >> 2) + i * (TC_XF_THREADS / 4);
            const int b = (m < p.M ? m : p.M - 1) / p.rows_per_sample;
            tmu[i] = __ldg(p.row_mean + b);
            trs[i] = __ldg(p.row_rstd + b);
          }
        }
        mbar_wait(&full[stage], (it / NST) & 1);
        uint8_t* st = sA + stage * RING_STAGE;
#pragma unroll
        for (int i = 0; i < TC_XF_IT; ++i) {
          const int c = tt + i * TC_XF_THREADS;
          const int row = c >> 2, ch = c & 3;
          const int k = k0 + ch * 8;
          const uint32_t off = (uint32_t)(row * 64 + ((ch ^ ((row >> 1) & 3)) << 4));  // 64-byte swizzle (TMA == wgmma layout)
          uint4* pa = reinterpret_cast<uint4*>(st + off);
          float f[8], q0[8], q1[8];
          unpack8(*pa, f);
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
          } else if (AMODE == CVB_A_BNB) {
            float y[8], q2[8];
            unpack8(*reinterpret_cast<const uint4*>(st + TC_STAGE + off), y);
            *reinterpret_cast<float4*>(q2) = *reinterpret_cast<const float4*>(sP + 2 * Kpad + k);
            *reinterpret_cast<float4*>(q2 + 4) = *reinterpret_cast<const float4*>(sP + 2 * Kpad + k + 4);
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = fmaf(q0[e], f[e], fmaf(q1[e], y[e], q2[e]));
          }
          // rows beyond M must stay exactly zero (their accumulators would otherwise pollute the statistics)
          *pa = (m0 + row < p.M) ? pack8(f) : make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async();  // generic-proxy writes above -> visible to the tensor core's async-proxy reads
        __syncwarp();
        if (lane == 0) mbar_arrive(&ready[stage]);
      }
    }
  } else {
    // ===================================================== consumer warpgroups: MMA, then the epilogue on the accumulator registers
    const int et = tid;                       // 0..TC_EPI_THREADS-1
    const int wg = tid >> 7;                  // channel half of the tile
    const int r0 = wg * 64 + ((tid & 127) >> 5) * 16 + (lane >> 2);  // local channel of acc[4j + {0,1}]; r0 + 8 holds acc[4j + {2,3}]
    const int pc = 2 * (lane & 3);            // pixel column of acc[4j] within the 8-column block j
    int chn[2];
    bool ch_ok[2];
    float bias[2], ep0[2], ep1[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      chn[h] = n0 + r0 + 8 * h;
      ch_ok[h] = chn[h] < p.N;
      bias[h] = (ch_ok[h] && p.bias) ? __ldg(p.bias + chn[h]) : 0.f;
      ep0[h] = ((EPI == TEPI_SILU_BWD || EPI == TEPI_GN_BWD) && ch_ok[h] && p.e_p0) ? __ldg(p.e_p0 + chn[h]) : 1.f;
      ep1[h] = (EPI == TEPI_SILU_BWD && ch_ok[h] && p.e_p1) ? __ldg(p.e_p1 + chn[h]) : 0.f;
    }
    constexpr bool has_aux = (EPI != TEPI_STORE);
    const bf16* __restrict__ AUX = static_cast<const bf16*>(EPI == TEPI_STORE_R ? p.R : p.Y);
    const int ldaux = EPI == TEPI_STORE_R ? p.ldr : p.ldy;
    const bool want_samp = (p.samp_sum != nullptr) && (EPI != TEPI_GN_BWD);  // GN_BWD: the sample sums come from the workspace finalize
    const bool lin_bwd = (p.e_mode == CVB_E_LIN_BWD);  // SiLU-backward epilogue without the activation factor (BatchNorm with no act)
    const int rps = p.rows_per_sample > 0 ? p.rows_per_sample : 1;
    float cs[2] = {0.f, 0.f}, cq[2] = {0.f, 0.f};  // statistics of this thread's two channels over its pixels of all tiles of the CTA
    bf16* __restrict__ Cg = static_cast<bf16*>(p.C);
    constexpr int CGS = TC_BN / 8;
    const uint32_t w_off = (uint32_t)wg * 64 * 64;  // this warpgroup's 64 weight rows (8 swizzle atoms of 512 B)

    auto issue_aux = [&](int j) {
      const int m0 = ((int)blockIdx.y + j * (int)gridDim.y) * TC_BM;
      for (int c = et; c < TC_BM * CGS; c += TC_EPI_THREADS) {
        const int row = c / CGS, cgc = c % CGS;
        const int m = m0 + row, n = n0 + cgc * 8;
        const bool ok = (m < p.M) && (n < p.N);
        cp_async16(smem_u32(sO + row * (TC_LDO * 2) + cgc * 16), AUX + (ok ? (size_t)m * ldaux + n : 0), ok);
      }
      cp_async_commit();
    };
    if (has_aux && my_tiles > 0) issue_aux(0);
    if (WRES) mbar_wait(&wbar, 0);

    float acc[64];
    int it = 0;
    for (int j = 0; j < my_tiles; ++j) {
      const int m0 = ((int)blockIdx.y + j * (int)gridDim.y) * TC_BM;
      for (int kt = 0; kt < KT; ++kt, ++it) {
        const int stage = it % NST;
        mbar_wait(XF ? &ready[stage] : &full[stage], (it / NST) & 1);  // landed (and transformed in place)
        const uint32_t aa = smem_u32(sA + stage * RING_STAGE);
        const uint32_t wa = (WRES ? smem_u32(sW + kt * TC_WBLK) : aa + A_BYTES) + w_off;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) wgmma_m64n128<0, 0>(acc, desc_sw64(wa + k * 32), desc_sw64(aa + k * 32), (kt | k) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have read their stage
        if (kt > 0 && (tid & 127) == 0) mbar_arrive(&empty[(it - 1) % NST]);
      }
      wgmma_wait<0>();
      wgmma_reg_fence<64>(acc);
      if ((tid & 127) == 0) mbar_arrive(&empty[(it - 1) % NST]);

      if (has_aux) {
        cp_async_wait<0>();
        epi_bar_sync();  // aux tile visible to all epilogue threads
      }
      const bool full_tile = (m0 + TC_BM <= p.M);  // rows >= M have zero A rows; only their bias must be masked (last tile)
      float gs[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, gq[2][2] = {{0.f, 0.f}, {0.f, 0.f}};  // GN_BWD: per channel, per 64-pixel half
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        bf16* so = reinterpret_cast<bf16*>(sO) + r0 + 8 * h;
        if (full_tile && !has_aux) {
          // hot path (conv -> BN statistics).  The BatchNorm sums are taken from the fp32 values (before bf16 rounding): the
          // rounding error averages out over the >= 128 pixels of the tile.
#pragma unroll
          for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v = acc[4 * jb + 2 * h + e] + bias[h];
              so[(8 * jb + pc + e) * TC_LDO] = __float2bfloat16_rn(v);
              cs[h] += v;
              cq[h] = fmaf(v, v, cq[h]);
            }
          }
        } else {
#pragma unroll
          for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int i = 8 * jb + pc + e;  // pixel within the tile
              float v = acc[4 * jb + 2 * h + e] + ((full_tile || m0 + i < p.M) ? bias[h] : 0.f);
              float y = 0.f;
              if (has_aux) y = __bfloat162float(so[i * TC_LDO]);
              if (EPI == TEPI_STORE_R) v += y;
              if (EPI == TEPI_SILU_BWD && !lin_bwd) v *= silu_grad_f(fmaf(ep0[h], y, ep1[h]));
              if (EPI == TEPI_GN_BWD) {
                // GroupNorm backward, phase 1 in sum form: per (sample, channel) A = sum v, Bx = sum v*x (raw x); everything else
                // (dgamma, dbeta, per-sample sums of g and g*xhat) is linear in A and Bx and is derived by the finalize kernel
                gs[h][jb >> 3] += v;
                gq[h][jb >> 3] = fmaf(v, y, gq[h][jb >> 3]);
                so[i * TC_LDO] = __float2bfloat16_rn(v * ep0[h]);
              } else {
                const bf16 vb = __float2bfloat16_rn(v);
                so[i * TC_LDO] = vb;
                const float vr = __bfloat162float(vb);  // statistics of the STORED values
                cs[h] += vr;
                cq[h] = fmaf(vr, EPI == TEPI_SILU_BWD ? y : vr, cq[h]);
              }
            }
          }
        }
      }
      if (EPI == TEPI_GN_BWD) {  // a 64-pixel half tile never straddles samples (rows_per_sample % 64 == 0, checked on the host)
        const int nsamples = (p.M + rps - 1) / rps;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            float a = gs[h][hf], bx = gq[h][hf];
            a += __shfl_xor_sync(0xffffffffu, a, 1);
            a += __shfl_xor_sync(0xffffffffu, a, 2);
            bx += __shfl_xor_sync(0xffffffffu, bx, 1);
            bx += __shfl_xor_sync(0xffffffffu, bx, 2);
            const int mh = m0 + hf * 64;
            if ((lane & 3) == 0 && ch_ok[h] && mh < p.M) {
              double* wsA = p.gn_ws + (size_t)(mh / rps) * p.N + chn[h];
              atomicAdd(wsA, (double)a);
              atomicAdd(wsA + (size_t)nsamples * p.N, (double)bx);
            }
          }
        }
      }
      epi_bar_sync();  // staged tile complete
      const int first_sample = m0 / rps;
      for (int c = et; c < TC_BM * CGS; c += TC_EPI_THREADS) {
        const int row = c / CGS, cgc = c % CGS;
        const int m = m0 + row, n = n0 + cgc * 8;
        const uint4 u = *reinterpret_cast<const uint4*>(sO + row * (TC_LDO * 2) + cgc * 16);
        if (m < p.M && n < p.N) stg16(Cg + (size_t)m * p.ldc + n, u);
        if (want_samp) {
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
            atomicAdd(&s_samp[0][m / rps - first_sample], (double)sv);
            atomicAdd(&s_samp[1][m / rps - first_sample], (double)sq);
          }
        }
      }
      epi_bar_sync();  // staging tile free again (and s_samp complete)
      if (want_samp) {
        const int mlast = min(m0 + TC_BM, p.M) - 1;
        const int nsamp = mlast / rps - first_sample + 1;
        if (et < nsamp) {
          atomicAdd(p.samp_sum + first_sample + et, s_samp[0][et]);
          atomicAdd(p.samp_sq + first_sample + et, s_samp[1][et]);
          s_samp[0][et] = 0.0;
          s_samp[1][et] = 0.0;
        }
      }
      if (has_aux && j + 1 < my_tiles) issue_aux(j + 1);
    }
    if (EPI != TEPI_GN_BWD) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {  // the four threads of a quad share a channel
        float s = cs[h], q = cq[h];
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        q += __shfl_xor_sync(0xffffffffu, q, 1);
        q += __shfl_xor_sync(0xffffffffu, q, 2);
        if (p.col_sum && ch_ok[h] && (lane & 3) == 0) {
          atomicAdd(p.col_sum + chn[h], (double)s);
          atomicAdd(p.col_sq + chn[h], (double)q);
        }
      }
    }
  }
}

template <int AMODE, int EPI, bool WRES>
int launch_tc_impl(const cvb_gemm_args& a, cudaStream_t st, size_t fixed, int stage_bytes) {
  const size_t budget = (size_t)216 * 1024;
  int nst = (int)((budget - fixed) / stage_bytes);
  if (nst > TC_MAX_STAGES) nst = TC_MAX_STAGES;
  const size_t smem = fixed + (size_t)nst * stage_bytes;
  static bool attr = false;
  if (!attr) {
    CVB_CUDA(cudaFuncSetAttribute(pw_gemm_tc_kernel<AMODE, EPI, WRES>, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));
    attr = true;
  }
  const int n_tiles = (a.N + TC_BN - 1) / TC_BN, m_tiles = (a.M + TC_BM - 1) / TC_BM;
  // one persistent CTA per SM, never more CTAs than SMs: rounding UP (e.g. 3 N tiles x 45 = 135 CTAs on 132 SMs) would put a few CTAs
  // into a second wave and double the time of the layer
  int gy = cvb_num_sms() / n_tiles;
  if (gy > m_tiles) gy = m_tiles;
  if (gy < 1) gy = 1;
  CUtensorMap tmA, tmA2, tmW;
  if (cvb_make_tmap_2d_k32(&tmA, a.A, a.M, a.K, a.lda, TC_BM)) return 1;
  if (cvb_make_tmap_2d_k32(&tmA2, AMODE == CVB_A_BNB ? a.A2 : a.A, a.M, a.K, AMODE == CVB_A_BNB ? a.lda2 : a.lda, TC_BM)) return 1;
  if (cvb_make_tmap_2d_k32(&tmW, a.W, a.N, a.K, a.ldw, TC_BN)) return 1;
  dim3 grid(n_tiles, gy);
  const int threads = TC_THREADS + XfCfg<AMODE>::THREADS;
  CVB_CUDA(cvb_launch(pw_gemm_tc_kernel<AMODE, EPI, WRES>, grid, threads, smem, st, tmA, tmA2, tmW, a, nst));
  CVB_LAUNCH_CHECK();
  return 0;
}

template <int AMODE, int EPI>
int launch_tc(const cvb_gemm_args& a, cudaStream_t st) {
  const int KT = (a.K + TC_BK - 1) / TC_BK;
  const int nvec = (AMODE == CVB_A_AFF || AMODE == CVB_A_AFF_SILU || AMODE == CVB_A_GN) ? 2 : (AMODE == CVB_A_BNB ? 3 : 0);
  const int a_bytes = (AMODE == CVB_A_BNB ? 2 : 1) * TC_STAGE;
  const size_t stagebuf = (size_t)TC_BM * TC_LDO * 2 + (size_t)nvec * KT * TC_BK * 4 + 1024;
  const size_t panel = (size_t)KT * TC_WBLK;
  if (panel + stagebuf + 6 * (size_t)a_bytes <= (size_t)216 * 1024) return launch_tc_impl<AMODE, EPI, true>(a, st, panel + stagebuf, a_bytes);
  return launch_tc_impl<AMODE, EPI, false>(a, st, stagebuf, a_bytes + TC_WBLK);  // large K: weight k-blocks ride the ring
}

// GroupNorm backward, phase 1 finalize: from A[b,c] = sum_m v, Bx[b,c] = sum_m v*x over the pixels of sample b
//   dbeta[c] += sum_b A;  dgamma[c] += sum_b t,  t = rstd_b (Bx - mean_b A) = sum_m v*xhat;   sum g = sum_c gamma_c A;   sum g*xhat = sum_c gamma_c t
// Blocks [0, B) take the per-sample sums, blocks [B, B + ceil(N / 16)) the per-channel ones.  A and t are full fp64 values, so the channel sums
// add the samples in a fixed order (an fp64 atomic per sample would round differently depending on which block arrives first).
__global__ void __launch_bounds__(128) gn_bwd_ws_finalize_kernel(const double* __restrict__ ws, const float* __restrict__ mean,
                                                                  const float* __restrict__ rstd, const float* __restrict__ gamma, int B, int N,
                                                                  double* col_sum, double* col_sq, double* samp_sum, double* samp_sq) {
  pdl_wait();
  pdl_trigger();
  __shared__ double s_red[2][4];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (b >= B) {  // 16 channels per block, 8 strided sample groups per channel, combined in group order
    __shared__ double s_col[2][8][16];
    const int cl = tid & 15, sg = tid >> 4, c = (b - B) * 16 + cl;
    double sa = 0.0, st = 0.0;
    if (c < N) {
#pragma unroll 4
      for (int s = sg; s < B; s += 8) {
        const double A = ws[(size_t)s * N + c], Bx = ws[((size_t)B + s) * N + c];
        sa += A;
        st += (double)rstd[s] * (Bx - (double)mean[s] * A);
      }
    }
    s_col[0][sg][cl] = sa;
    s_col[1][sg][cl] = st;
    __syncthreads();
    if (sg == 0 && c < N) {
      for (int g = 1; g < 8; ++g) { sa += s_col[0][g][cl]; st += s_col[1][g][cl]; }
      col_sum[c] += sa;
      col_sq[c] += st;
    }
    return;
  }
  const double mu = (double)mean[b], rs = (double)rstd[b];
  double sg = 0.0, sgx = 0.0;
  for (int c = tid; c < N; c += 128) {
    const double A = ws[(size_t)b * N + c], Bx = ws[((size_t)B + b) * N + c];
    const double t = rs * (Bx - mu * A);
    const double gm = gamma ? (double)gamma[c] : 1.0;
    sg += gm * A;
    sgx += gm * t;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sg += __shfl_xor_sync(0xffffffffu, sg, o);
    sgx += __shfl_xor_sync(0xffffffffu, sgx, o);
  }
  if ((tid & 31) == 0) { s_red[0][tid >> 5] = sg; s_red[1][tid >> 5] = sgx; }
  __syncthreads();
  if (tid == 0 && samp_sum) {
    atomicAdd(samp_sum + b, s_red[0][0] + s_red[0][1] + s_red[0][2] + s_red[0][3]);
    atomicAdd(samp_sq + b, s_red[1][0] + s_red[1][1] + s_red[1][2] + s_red[1][3]);
  }
}

template <int AMODE>
int launch_tc_gn_bwd(const cvb_gemm_args& a, cudaStream_t st) {
  int rc = launch_tc<AMODE, TEPI_GN_BWD>(a, st);
  if (rc != 0) return rc;
  const int B = (a.M + a.rows_per_sample - 1) / a.rows_per_sample;
  const int col_blocks = a.col_sum ? (a.N + 15) / 16 : 0;
  CVB_CUDA(cvb_launch(gn_bwd_ws_finalize_kernel, B + col_blocks, 128, 0, st, static_cast<const double*>(a.gn_ws), a.row_mean, a.row_rstd, a.e_p0, B, a.N, a.col_sum,
                      a.col_sq, a.samp_sum, a.samp_sq));
  CVB_LAUNCH_CHECK();
  return 0;
}

template <int AMODE>
int dispatch_tc_epi(const cvb_gemm_args& a, cudaStream_t st) {
  if (a.e_mode == CVB_E_GN_BWD && a.gn_ws && a.rows_per_sample % (TC_BM / 2) == 0 && !a.bias && (AMODE == CVB_A_RAW || AMODE == CVB_A_BNB))
    return launch_tc_gn_bwd<AMODE == CVB_A_BNB ? CVB_A_BNB : CVB_A_RAW>(a, st);
  if (a.e_mode == CVB_E_STORE) return a.R ? launch_tc<AMODE, TEPI_STORE_R>(a, st) : launch_tc<AMODE, TEPI_STORE>(a, st);
  if ((a.e_mode == CVB_E_SILU_BWD || a.e_mode == CVB_E_LIN_BWD) && (AMODE == CVB_A_RAW || AMODE == CVB_A_BNB)) return launch_tc<AMODE == CVB_A_BNB ? CVB_A_BNB : CVB_A_RAW, TEPI_SILU_BWD>(a, st);
  return -1;
}

}  // namespace

// Returns -1 when the shape / mode is not handled by the wgmma kernel (caller uses the mma.sync kernel), 0 on success, > 0 on error.
// any_n: take narrow / ragged N too (the mma.sync kernel cannot hold this K).
int cvb_pw_gemm_tc(const cvb_gemm_args& a, cudaStream_t st, bool any_n) {
  // a CTA computes 128 output channels: narrow layers would idle most of them -> mma.sync kernel
  if (!any_n && (a.N < 96 || (a.N % 128 != 0 && a.N % 128 < 64 && a.N < 256))) return -1;  // narrow / ragged N would leave most of a 128-channel tile idle
  switch (a.a_mode) {
    case CVB_A_RAW: return dispatch_tc_epi<CVB_A_RAW>(a, st);
    case CVB_A_AFF: return dispatch_tc_epi<CVB_A_AFF>(a, st);
    case CVB_A_AFF_SILU: return dispatch_tc_epi<CVB_A_AFF_SILU>(a, st);
    case CVB_A_SILU: return dispatch_tc_epi<CVB_A_SILU>(a, st);
    case CVB_A_GN: return dispatch_tc_epi<CVB_A_GN>(a, st);
    case CVB_A_BNB: return dispatch_tc_epi<CVB_A_BNB>(a, st);
    default: return -1;
  }
}
