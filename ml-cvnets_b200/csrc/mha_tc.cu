// wgmma / TMA multi-head attention core for head_dim == 64, S <= 256 (ViT-B 197 x 64), sm_90a.
// Same contract as mha.cu (cvnets/layers/multi_head_attention.py:187-237): packed projection in, O / LSE out, dQKV in the backward.
// Key-padding masks only: the router in mha.cu sends heads with an additive mask to the mma.sync kernels.
//
// Every operand of a head -- Q, K, V, dO [rows x 64 bf16] -- is ONE TMA box [64 cols x rows] with 128-byte swizzle.  That shared-memory
// image (128-byte rows, 8-row swizzle atoms of 1 KB) is at the same time
//   * the canonical K-major  SWIZZLE_128B wgmma operand  (rows = M/N, the 64 channels = K)        -> S = Q K^T, dP^T = V dO^T
//   * the canonical MN-major SWIZZLE_128B wgmma operand  (the 64 channels = N, rows = K)           -> O = P V, dV = P^T dO, dK = dS^T Q, dQ = dS K
// so nothing is transposed or loaded twice.  A whole score row (S <= 256) stays in the accumulator registers of its warpgroup: the
// softmax needs no second pass over memory, and P / dS^T go straight from those registers into the A operand of the next wgmma.
//
// Forward, one CTA per (sample, head, 128-query tile): two warpgroups of 64 query rows each; thread 0 issues the TMA loads.
// Backward, one CTA per (sample, head): the two warpgroups take alternate 64-key blocks; per (key block, 64-query block)
//   S^T = K Q^T, dP^T = V dO^T (registers) -> P^T, dS^T -> dV += P^T dO, dK += dS^T Q (register A operands), dQ_q += dS K (dS^T staged
//   in shared memory, fp32 dQ accumulated in shared memory across the key blocks of both warpgroups)
#include "mha_wgmma.cuh"

namespace {

// byte offset of the 16-byte chunk `ch` (0..7) of row `row` inside a [rows x 64 ch] SWIZZLE_128B image
__device__ __forceinline__ uint32_t sw128(int row, int ch) { return static_cast<uint32_t>(row * 128 + ((ch ^ (row & 7)) << 4)); }
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

// ------------------------------------------------------------------------------------------------------------- forward
constexpr int FW_THREADS = 256;

__global__ void __launch_bounds__(FW_THREADS, 1)
    mha_tc_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV, int S, int NCH, int H, int NQT, float scale,
                      const uint8_t* __restrict__ kpm, bf16* __restrict__ O, int ldo, float* __restrict__ LSE) {
  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7;
  int bid = blockIdx.x;
  const int qt = bid % NQT;
  bid /= NQT;
  const int h = bid % H, b = bid / H;
  const int C = H * 64;
  const int Sk = NCH * 64;  // key rows loaded (zero-filled past the tensor)

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;                 // [128 q][64]
  uint8_t* sK = sQ + 2 * BOX64;       // [Sk t][64]
  uint8_t* sV = sK + Sk * 128;        // [Sk t][64]
  __shared__ __align__(8) uint64_t bar_qk, bar_v;

  if (tid == 0) {
    mbar_init(&bar_qk, 1);
    mbar_init(&bar_v, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  if (tid == 0) {
    const int row0 = b * S;
    mbar_expect_tx(&bar_qk, (uint32_t)(2 * BOX64 + Sk * 128));
    tma_load_2d(sQ, &tmQ, &bar_qk, h * 64, row0 + qt * 128);
    tma_load_2d(sK, &tmKV, &bar_qk, C + h * 64, row0);
    mbar_expect_tx(&bar_v, (uint32_t)(Sk * 128));
    tma_load_2d(sV, &tmKV, &bar_v, 2 * C + h * 64, row0);
  }

  const int rl = ((tid & 127) >> 5) * 16 + (lane >> 2);  // query row (within the warpgroup's 64) of acc[4j + {0,1}]; + 8 for {2,3}
  const int q0 = qt * 128 + wg * 64;
  const float sc2 = scale * LOG2E;
  const uint32_t aQ = smem_u32(sQ) + wg * BOX64, aK = smem_u32(sK), aV = smem_u32(sV);

  // ---- S = Q K^T, 64-key chunks
  float sacc[4][32];
  mbar_wait(&bar_qk, 0);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < 4; ++c)
    if (c < NCH) {
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(sacc[c], desc_k(aQ + k * 32), desc_k(aK + c * BOX64 + k * 32), k ? 1u : 0u);
    }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < 4; ++c) wgmma_reg_fence<32>(sacc[c]);

  // ---- softmax in the exp2 domain; a row is spread over the 4 threads of a quad
  float m[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
  for (int c = 0; c < 4; ++c)
    if (c < NCH) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int hh = (i >> 1) & 1, q = q0 + rl + 8 * hh, t = c * 64 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        float v = -CUDART_INF_F;
        if (t < S) {
          v = sacc[c][i] * sc2;
          if (kpm) v += mask_add(nullptr, kpm, b, S, q, t);
        }
        sacc[c][i] = v;
        m[hh] = fmaxf(m[hh], v);
      }
    }
  float l[2] = {0.f, 0.f}, msafe[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    m[hh] = fmaxf(m[hh], __shfl_xor_sync(0xffffffffu, m[hh], 1));
    m[hh] = fmaxf(m[hh], __shfl_xor_sync(0xffffffffu, m[hh], 2));
    msafe[hh] = (m[hh] == -CUDART_INF_F) ? 0.f : m[hh];  // a fully masked row must not produce inf - inf
  }
#pragma unroll
  for (int c = 0; c < 4; ++c)
    if (c < NCH) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int hh = (i >> 1) & 1;
        const float pv = ex2(sacc[c][i] - msafe[hh]);
        sacc[c][i] = pv;
        l[hh] += pv;
      }
    }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
  }

  // ---- O = P V (P as bf16 register operand, V MN-major)
  float oacc[32];
  mbar_wait(&bar_v, 0);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < 4; ++c)
    if (c < NCH) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t a[4];
        to_a_frag(sacc[c], kk, a);
        wgmma_m64n64_rs<1>(oacc, a, desc_mn(aV + (c * 64 + kk * 16) * 128), (c | kk) ? 1u : 0u);
      }
    }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_reg_fence<32>(oacc);

  // ---- epilogue: O / l (a fully masked row gives 0 * inf = NaN, like softmax over an all -inf row in the reference), LSE
  const float inv[2] = {1.0f / l[0], 1.0f / l[1]};
#pragma unroll
  for (int i = 0; i < 32; ++i) oacc[i] *= inv[(i >> 1) & 1];
  store_acc(O + (size_t)b * S * ldo + h * 64, ldo, oacc, 1.0f, q0, S);
  if ((lane & 3) == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q = q0 + rl + 8 * hh;
      if (q < S) LSE[((size_t)b * H + h) * S + q] = m[hh] + log2f(l[hh]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ backward
constexpr int BW_THREADS = 256;

__global__ void __launch_bounds__(BW_THREADS, 1)
    mha_tc_bwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO, const bf16* __restrict__ O,
                      const bf16* __restrict__ DO, int ldo, const float* __restrict__ LSE, int S, int H, int NB, float scale,
                      const uint8_t* __restrict__ kpm, bf16* __restrict__ DQKV, int lddq) {
  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7;
  const int h = blockIdx.x % H, b = blockIdx.x / H;
  const int C = H * 64;
  const int R = NB * 64;  // rows of every operand image

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + R * 128;
  uint8_t* sV = sK + R * 128;
  uint8_t* sdO = sV + R * 128;
  uint8_t* sdST = sdO + R * 128;                              // per warpgroup: dS^T [64 keys][64 queries]
  float* sdQ = reinterpret_cast<float*>(sdST + 2 * BOX64);    // fp32 [R][64]
  float* sLSE = sdQ + R * 64;                                 // [R]
  float* sD = sLSE + R;                                       // [R]: D = sum_c dO O
  __shared__ __align__(8) uint64_t bar_ld;

  if (tid == 0) {
    mbar_init(&bar_ld, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  if (tid == 0) {
    const int row0 = b * S;
    mbar_expect_tx(&bar_ld, (uint32_t)(4 * R * 128));
    tma_load_2d(sQ, &tmQKV, &bar_ld, h * 64, row0);
    tma_load_2d(sK, &tmQKV, &bar_ld, C + h * 64, row0);
    tma_load_2d(sV, &tmQKV, &bar_ld, 2 * C + h * 64, row0);
    tma_load_2d(sdO, &tmDO, &bar_ld, h * 64, row0);
  }
  for (int i = tid; i < R * 64; i += BW_THREADS) sdQ[i] = 0.f;
  for (int q = tid; q < R; q += BW_THREADS) {
    float lv = 0.f, d = 0.f;
    if (q < S) {
      lv = LSE[((size_t)b * H + h) * S + q];
      const bf16* orow = O + ((size_t)b * S + q) * ldo + h * 64;
      const bf16* drow = DO + ((size_t)b * S + q) * ldo + h * 64;
#pragma unroll
      for (int ch = 0; ch < 8; ++ch) {
        float a[8], c[8];
        unpack8(ldg16(orow + ch * 8), a);
        unpack8(ldg16(drow + ch * 8), c);
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(a[e], c[e], d);
      }
    }
    sLSE[q] = lv;
    sD[q] = d;
  }
  __syncthreads();
  mbar_wait(&bar_ld, 0);

  const int rl = ((tid & 127) >> 5) * 16 + (lane >> 2);  // key row (within the block) of acc[4j + {0,1}]; + 8 for {2,3}
  const float sc2 = scale * LOG2E;
  const uint32_t aQ = smem_u32(sQ), aK = smem_u32(sK), aV = smem_u32(sV), aDO = smem_u32(sdO), aDS = smem_u32(sdST) + wg * BOX64;
  uint8_t* my_dST = sdST + wg * BOX64;
  bf16* dbase = DQKV + (size_t)b * S * lddq + h * 64;

  for (int kb = wg; kb < NB; kb += 2) {
    float dk[32], dv[32];
    for (int qb = 0; qb < NB; ++qb) {
      float st[32], dpt[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(st, desc_k(aK + kb * BOX64 + k * 32), desc_k(aQ + qb * BOX64 + k * 32), k ? 1u : 0u);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(dpt, desc_k(aV + kb * BOX64 + k * 32), desc_k(aDO + qb * BOX64 + k * 32), k ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence<32>(st);
      wgmma_reg_fence<32>(dpt);
      // P^T = exp2(s sc2 + mask - lse), dS^T = P^T (dP^T - D); zero outside the sequence and for masked keys
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int t = kb * 64 + rl + 8 * ((i >> 1) & 1), q = qb * 64 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        float pv = 0.f, dv2 = 0.f;
        if (q < S && t < S) {
          float v = fmaf(st[i], sc2, -sLSE[q]);
          if (kpm) v += mask_add(nullptr, kpm, b, S, q, t);
          pv = ex2(v);
          dv2 = pv * (dpt[i] - sD[q]);
          if (pv == 0.f) dv2 = 0.f;  // masked keys: exactly zero whatever dP holds
        }
        st[i] = pv;
        dpt[i] = dv2;
      }
      // dS^T as bf16 [64 keys][64 queries] SWIZZLE_128B image: the MN-major A operand of dQ = dS K
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = rl + 8 * hh;
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<uint32_t*>(my_dST + sw128(row, j) + 4 * (lane & 3)) = pack_bf162(dpt[4 * j + 2 * hh], dpt[4 * j + 2 * hh + 1]);
      }
      fence_proxy_async();
      wg_bar(wg);
      float dq[32];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // reduction over the 64 queries of the block
        uint32_t a[4];
        to_a_frag(st, kk, a);
        wgmma_m64n64_rs<1>(dv, a, desc_mn(aDO + (qb * 64 + kk * 16) * 128), (qb | kk) ? 1u : 0u);
        to_a_frag(dpt, kk, a);
        wgmma_m64n64_rs<1>(dk, a, desc_mn(aQ + (qb * 64 + kk * 16) * 128), (qb | kk) ? 1u : 0u);
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)  // reduction over the 64 keys of the block
        wgmma_m64n64<1, 1>(dq, desc_mn(aDS + kk * 2048), desc_mn(aK + (kb * 64 + kk * 16) * 128), kk ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_reg_fence<32>(dv);
      wgmma_reg_fence<32>(dk);
      wgmma_reg_fence<32>(dq);
#pragma unroll
      for (int i = 0; i < 32; ++i)  // dQ rows = queries of the block, columns = channels
        atomicAdd(sdQ + (qb * 64 + rl + 8 * ((i >> 1) & 1)) * 64 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1), dq[i]);
      wg_bar(wg);  // every thread's reads of the dS^T image are complete before it is rewritten
    }
    store_acc(dbase + C, lddq, dk, scale, kb * 64, S);
    store_acc(dbase + 2 * C, lddq, dv, 1.0f, kb * 64, S);
  }
  __syncthreads();
  for (int i = tid; i < S * 8; i += BW_THREADS) {  // dQ: 8 chunks of 8 channels per query row
    const int q = i >> 3, c8 = (i & 7) * 8;
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = sdQ[q * 64 + c8 + e] * scale;
    stg16(dbase + (size_t)q * lddq + c8, pack8(f));
  }
}

}  // namespace

int cvb_mha_fwd_tc(const void* QKV, int ldq, int B, int S, int H, float scale, const unsigned char* kpm, void* O, int ldo, float* LSE, cudaStream_t st) {
  const int NCH = (S + 63) / 64;
  const int NQT = (S + 127) / 128;
  CUtensorMap tmQ, tmKV;
  if (cvb_make_tmap_2d(&tmQ, QKV, (int64_t)B * S, 3 * H * 64, ldq, 128, 64)) return 1;
  if (cvb_make_tmap_2d(&tmKV, QKV, (int64_t)B * S, 3 * H * 64, ldq, NCH * 64, 64)) return 1;
  const size_t smem = (size_t)2 * BOX64 + (size_t)2 * NCH * BOX64 + 1024;
  CVB_CUDA(cvb_smem_optin<mha_tc_fwd_kernel>(96 * 1024));
  CVB_CUDA(cvb_launch(mha_tc_fwd_kernel, B * H * NQT, FW_THREADS, smem, st, tmQ, tmKV, S, NCH, H, NQT, scale, kpm, static_cast<bf16*>(O), ldo, LSE));
  return 0;
}

int cvb_mha_bwd_tc(const void* QKV, int ldq, const void* O, const void* DO, int ldo, const float* LSE, int B, int S, int H, float scale,
                   const unsigned char* kpm, void* DQKV, int lddq, cudaStream_t st) {
  const int NB = (S + 63) / 64;
  const int R = NB * 64;
  CUtensorMap tmQKV, tmDO;
  if (cvb_make_tmap_2d(&tmQKV, QKV, (int64_t)B * S, 3 * H * 64, ldq, R, 64)) return 1;
  if (cvb_make_tmap_2d(&tmDO, DO, (int64_t)B * S, H * 64, ldo, R, 64)) return 1;
  // Q, K, V, dO images + two dS^T images + fp32 dQ + LSE / D
  const size_t smem = (size_t)4 * R * 128 + 2 * BOX64 + (size_t)R * 64 * 4 + (size_t)2 * R * 4 + 1024;
  CVB_CUDA(cvb_smem_optin<mha_tc_bwd_kernel>(224 * 1024));
  CVB_CUDA(cvb_launch(mha_tc_bwd_kernel, B * H, BW_THREADS, smem, st, tmQKV, tmDO, static_cast<const bf16*>(O), static_cast<const bf16*>(DO), ldo, LSE, S,
                      H, NB, scale, kpm, static_cast<bf16*>(DQKV), lddq));
  return 0;
}
