// Multi-head self-attention core (cvnets/layers/multi_head_attention.py:135-239), forward and backward, sm_90a.
//
//   O[b, s, h*c + :] = softmax_t( scale * Q[b,h,s,:] . K[b,h,t,:] + attn_mask[b,s,t]  (-inf where key_padding_mask[b,t]) ) @ V[b,h,t,:]
//
// Q, K, V are strided views of the packed projection qkv[b*S + s, {0,1,2}*C + h*c + :] (the reference reshapes to [N,S,3,h,c],
// :148-153), O is written straight into the [N*S, C] layout out_proj consumes (:236) -- no transposes, no [N,h,S,T] score
// tensor in HBM (the reference materialises it twice, bf16 and fp32: 477 MB per ViT-B layer, SURVEY.md 8a a11).
// One CTA per (sample, head); the whole K / V (and Q, dO in the backward) of that head live in shared memory (S <= 256,
// head_dim in {16, 32, 64}: every hot-path config of SURVEY.md 8a: ViT-B 197x64, CLIP text 77x64, MobileViT-v1 256x16..).
// Tensor cores: mma.sync.m16n8k16 bf16 -> fp32 (the score tiles are 16 x 64 per warp: far below a wgmma tile), online softmax
// in the exp2 domain, probabilities kept in registers and re-used as the A operand of P.V.
// Backward = two passes without atomics: pass A owns query rows (dQ), pass B owns key rows (dK, dV); P is recomputed from the
// saved log-sum-exp.
#include "common.cuh"

#include <math_constants.h>

namespace {

constexpr float LOG2E = 1.4426950408889634f;

template <int HD>
struct MhaCfg {
  static constexpr int LD = HD + 8;       // smem row stride in elements (16-byte aligned rows, ldmatrix conflict-free)
  static constexpr int KS = HD / 16;      // k-steps over the head dim
  static constexpr int NT = HD / 8;       // n-tiles over the head dim
};

// cooperative load of one [S, hd] strided operand into smem rows of HD >= hd columns (zero fill past S and past hd).  hd == HD: 16-byte
// chunks; otherwise (MobileViT-v1 head dims 20 / 24 / 36 / 48 / 60, hd % 4 == 0) 8-byte chunks -- a head's columns start at h * hd, which
// is 8- but not 16-byte aligned -- with the pad columns zero-filled, so that the padded tiles contribute nothing to any product.
__device__ __forceinline__ void cp_async8(uint32_t smem_addr, const void* gptr, bool pred) {
  int sz = pred ? 8 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(smem_addr), "l"(gptr), "r"(sz));
}
template <int HD>
__device__ __forceinline__ void load_rows(bf16* dst, const bf16* src, int ld, int S, int Sp, int hd, int tid, int nthreads) {
  constexpr int LD = MhaCfg<HD>::LD;
  if (hd == HD) {
    constexpr int CH = HD / 8;
    for (int idx = tid; idx < Sp * CH; idx += nthreads) {
      const int row = idx / CH, ch = idx % CH;
      const bool ok = row < S;
      cp_async16(smem_u32(dst + row * LD + ch * 8), src + (ok ? (size_t)row * ld + ch * 8 : 0), ok);
    }
  } else if (hd % 4 == 0) {
    constexpr int CH = HD / 4;
    for (int idx = tid; idx < Sp * CH; idx += nthreads) {
      const int row = idx / CH, ch = idx % CH;
      const bool ok = row < S && ch * 4 < hd;
      cp_async8(smem_u32(dst + row * LD + ch * 4), src + (ok ? (size_t)row * ld + ch * 4 : 0), ok);
    }
  } else {  // even head dims that are not multiples of 4 (MobileViT-XS: 120 / 4 = 30): 4-byte chunks
    constexpr int CH = HD / 2;
    for (int idx = tid; idx < Sp * CH; idx += nthreads) {
      const int row = idx / CH, ch = idx % CH;
      const bool ok = row < S && ch * 2 < hd;
      const int sz = ok ? 4 : 0;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(smem_u32(dst + row * LD + ch * 2)), "l"(src + (ok ? (size_t)row * ld + ch * 2 : 0)),
                   "r"(sz));
    }
  }
}

// scores of one 16 x 64 block: acc[nt][4] = A(16 x HD, fragments afr) . B^T, B = 64 rows of `sB` starting at row r0 (stored [row][HD])
template <int HD>
__device__ __forceinline__ void qk_block(float (*acc)[4], const uint32_t (*afr)[4], const bf16* sB, int r0, int lane) {
  constexpr int LD = MhaCfg<HD>::LD;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
#pragma unroll
  for (int ks = 0; ks < MhaCfg<HD>::KS; ++ks)
#pragma unroll
    for (int np = 0; np < 4; ++np) {  // pairs of n-tiles
      const int idx = lane >> 3;
      const int n = r0 + np * 16 + (idx >> 1) * 8 + (lane & 7);
      const int k = ks * 16 + (idx & 1) * 8;
      uint32_t b0, b1, b2, b3;
      ldmatrix_x4(smem_u32(sB + n * LD + k), b0, b1, b2, b3);
      mma_bf16_16816(acc[2 * np], afr[ks], b0, b1);
      mma_bf16_16816(acc[2 * np + 1], afr[ks], b2, b3);
    }
}
// out[NT][4] += P(16 x 64, packed fragments pfr[4][4]) . B, B = 64 rows of `sB` starting at row r0, stored [row = k][HD = n]
template <int HD>
__device__ __forceinline__ void pv_block(float (*out)[4], const uint32_t (*pfr)[4], const bf16* sB, int r0, int lane) {
  constexpr int LD = MhaCfg<HD>::LD;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)  // 16 rows of sB per step
#pragma unroll
    for (int np = 0; np < MhaCfg<HD>::NT / 2; ++np) {
      const int idx = lane >> 3;
      const int k = r0 + ks * 16 + (idx & 1) * 8 + (lane & 7);
      const int n = np * 16 + (idx >> 1) * 8;
      uint32_t b0, b1, b2, b3;
      ldmatrix_x4_trans(smem_u32(sB + k * LD + n), b0, b1, b2, b3);
      mma_bf16_16816(out[2 * np], pfr[ks], b0, b1);
      mma_bf16_16816(out[2 * np + 1], pfr[ks], b2, b3);
    }
}
template <int HD>
__device__ __forceinline__ void load_afrag(uint32_t (*afr)[4], const bf16* sA, int r0, int lane) {
  constexpr int LD = MhaCfg<HD>::LD;
#pragma unroll
  for (int ks = 0; ks < MhaCfg<HD>::KS; ++ks)
    ldmatrix_x4(smem_u32(sA + (r0 + (lane & 15)) * LD + ks * 16 + (lane >> 4) * 8), afr[ks][0], afr[ks][1], afr[ks][2], afr[ks][3]);
}
__device__ __forceinline__ void pack_p(uint32_t (*pfr)[4], const float (*acc)[4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    pfr[ks][0] = pack_bf162(acc[2 * ks][0], acc[2 * ks][1]);
    pfr[ks][1] = pack_bf162(acc[2 * ks][2], acc[2 * ks][3]);
    pfr[ks][2] = pack_bf162(acc[2 * ks + 1][0], acc[2 * ks + 1][1]);
    pfr[ks][3] = pack_bf162(acc[2 * ks + 1][2], acc[2 * ks + 1][3]);
  }
}
// additive mask (in the exp2 domain) of score element (q row, key col); -inf for padded / out-of-range keys
__device__ __forceinline__ float mask_term(const float* amask, const uint8_t* kpm, int b, int S, int q, int t) {
  if (t >= S) return -CUDART_INF_F;
  if (kpm && kpm[(size_t)b * S + t]) return -CUDART_INF_F;
  if (amask && q < S) return amask[((size_t)b * S + q) * S + t] * LOG2E;
  return 0.f;
}

// ------------------------------------------------------------------------------------------------------------- forward
template <int HD>
__global__ void __launch_bounds__(128) mha_fwd_kernel(const bf16* __restrict__ QKV, int ldq, int S, int H, float scale, const float* __restrict__ amask,
                                                      const uint8_t* __restrict__ kpm, bf16* __restrict__ O, int ldo, float* __restrict__ LSE, int hd) {
  constexpr int LD = MhaCfg<HD>::LD;
  constexpr int NT = MhaCfg<HD>::NT;
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int C = H * hd;
  const int Sp = (S + 63) / 64 * 64;
  bf16* sQ = reinterpret_cast<bf16*>(smem_raw);
  bf16* sK = sQ + Sp * LD;
  bf16* sV = sK + Sp * LD;
  const bf16* base = QKV + (size_t)b * S * ldq + h * hd;
  load_rows<HD>(sQ, base, ldq, S, Sp, hd, tid, 128);
  load_rows<HD>(sK, base + C, ldq, S, Sp, hd, tid, 128);
  load_rows<HD>(sV, base + 2 * C, ldq, S, Sp, hd, tid, 128);
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  const float sc2 = scale * LOG2E;
  const bool masked = (amask != nullptr) || (kpm != nullptr);

  for (int slab = warp; slab * 16 < S; slab += 4) {
    const int q0 = slab * 16;
    uint32_t qf[MhaCfg<HD>::KS][4];
    load_afrag<HD>(qf, sQ, q0, lane);
    float o[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
    float mrow[2] = {-CUDART_INF_F, -CUDART_INF_F}, lrow[2] = {0.f, 0.f};
    for (int kb = 0; kb < Sp; kb += 64) {
      float s[8][4];
      qk_block<HD>(s, qf, sK, kb, lane);
      const bool tail = masked || (kb + 64 > S);
      float bm[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = s[nt][e] * sc2;
          if (tail) v += mask_term(amask, kpm, b, S, q0 + g + (e >> 1) * 8, kb + nt * 8 + 2 * t4 + (e & 1));
          s[nt][e] = v;
          bm[e >> 1] = fmaxf(bm[e >> 1], v);
        }
      float corr[2], mnew[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 1));
        bm[r] = fmaxf(bm[r], __shfl_xor_sync(0xffffffffu, bm[r], 2));
        mnew[r] = fmaxf(mrow[r], bm[r]);
        const float msafe = (mnew[r] == -CUDART_INF_F) ? 0.f : mnew[r];  // a fully masked prefix must not produce inf - inf
        corr[r] = exp2f(mrow[r] - msafe);
        mrow[r] = mnew[r];
        mnew[r] = msafe;
      }
      float rs[2] = {0.f, 0.f};
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float pv = exp2f(s[nt][e] - mnew[e >> 1]);
          s[nt][e] = pv;
          rs[e >> 1] += pv;
        }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
        rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
        lrow[r] = lrow[r] * corr[r] + rs[r];
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        o[nt][0] *= corr[0]; o[nt][1] *= corr[0];
        o[nt][2] *= corr[1]; o[nt][3] *= corr[1];
      }
      uint32_t pf[4][4];
      pack_p(pf, s);
      pv_block<HD>(o, pf, sV, kb, lane);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = q0 + g + r * 8;
      if (q < S) {
        const float inv = 1.0f / lrow[r];  // a fully masked row gives 0 * inf = NaN, like softmax over an all -inf row in the reference
        bf16* orow = O + ((size_t)b * S + q) * ldo + h * hd;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
          if (nt * 8 + 2 * t4 < hd) *reinterpret_cast<uint32_t*>(orow + nt * 8 + 2 * t4) = pack_bf162(o[nt][2 * r] * inv, o[nt][2 * r + 1] * inv);
        if (t4 == 0) LSE[((size_t)b * H + h) * S + q] = mrow[r] + log2f(lrow[r]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ backward
template <int HD>
__global__ void __launch_bounds__(256) mha_bwd_kernel(const bf16* __restrict__ QKV, int ldq, const bf16* __restrict__ O, const bf16* __restrict__ DO,
                                                      int ldo, const float* __restrict__ LSE, int S, int H, float scale,
                                                      const float* __restrict__ amask, const uint8_t* __restrict__ kpm, bf16* __restrict__ DQKV,
                                                      int lddq, int hd) {
  constexpr int LD = MhaCfg<HD>::LD;
  constexpr int NT = MhaCfg<HD>::NT;
  constexpr int KS = MhaCfg<HD>::KS;
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int C = H * hd;
  const int Sp = (S + 63) / 64 * 64;
  bf16* sQ = reinterpret_cast<bf16*>(smem_raw);
  bf16* sK = sQ + Sp * LD;
  bf16* sV = sK + Sp * LD;
  bf16* sDO = sV + Sp * LD;
  float* sLse = reinterpret_cast<float*>(sDO + Sp * LD);
  float* sD = sLse + Sp;
  const bf16* base = QKV + (size_t)b * S * ldq + h * hd;
  const bf16* obase = O + (size_t)b * S * ldo + h * hd;
  const bf16* dobase = DO + (size_t)b * S * ldo + h * hd;
  load_rows<HD>(sQ, base, ldq, S, Sp, hd, tid, 256);
  load_rows<HD>(sK, base + C, ldq, S, Sp, hd, tid, 256);
  load_rows<HD>(sV, base + 2 * C, ldq, S, Sp, hd, tid, 256);
  load_rows<HD>(sDO, dobase, ldo, S, Sp, hd, tid, 256);
  cp_async_commit();
  // D[q] = sum_c dO[q,c] * O[q,c]  (softmax backward row term), lse of padded rows = +inf so that their P is exactly 0
  for (int q = tid; q < Sp; q += 256) {
    float d = 0.f;
    if (q < S) {
      if (hd == HD) {
#pragma unroll
        for (int ch = 0; ch < HD / 8; ++ch) {
          float a[8], c[8];
          unpack8(ldg16(obase + (size_t)q * ldo + ch * 8), a);
          unpack8(ldg16(dobase + (size_t)q * ldo + ch * 8), c);
#pragma unroll
          for (int e = 0; e < 8; ++e) d = fmaf(a[e], c[e], d);
        }
      } else {
        for (int c2 = 0; c2 < hd; c2 += 2) {
          const float2 a = unpack_bf162(*reinterpret_cast<const uint32_t*>(obase + (size_t)q * ldo + c2));
          const float2 c = unpack_bf162(*reinterpret_cast<const uint32_t*>(dobase + (size_t)q * ldo + c2));
          d = fmaf(a.x, c.x, fmaf(a.y, c.y, d));
        }
      }
    }
    sD[q] = d;
    sLse[q] = q < S ? LSE[((size_t)b * H + h) * S + q] : CUDART_INF_F;
  }
  cp_async_wait<0>();
  __syncthreads();
  const float sc2 = scale * LOG2E;
  const bool masked = (amask != nullptr) || (kpm != nullptr);
  bf16* dbase = DQKV + (size_t)b * S * lddq + h * hd;

  // ---- pass A: this warp owns 16 query rows -> dQ = scale * sum_t dS[q,t] K[t,:],  dS = P o (dP - D),  dP = dO V^T
  for (int slab = warp; slab * 16 < S; slab += 8) {
    const int q0 = slab * 16;
    uint32_t qf[KS][4], dof[KS][4];
    load_afrag<HD>(qf, sQ, q0, lane);
    load_afrag<HD>(dof, sDO, q0, lane);
    float dq[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) dq[nt][e] = 0.f;
    const float lse0 = sLse[q0 + g], lse1 = sLse[q0 + g + 8];
    const float d0 = sD[q0 + g], d1 = sD[q0 + g + 8];
    for (int kb = 0; kb < Sp; kb += 64) {
      float s[8][4], dp[8][4];
      qk_block<HD>(s, qf, sK, kb, lane);
      qk_block<HD>(dp, dof, sV, kb, lane);
      const bool tail = masked || (kb + 64 > S);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = s[nt][e] * sc2;
          if (tail) v += mask_term(amask, kpm, b, S, q0 + g + (e >> 1) * 8, kb + nt * 8 + 2 * t4 + (e & 1));
          const float pv = exp2f(v - ((e >> 1) ? lse1 : lse0));
          s[nt][e] = pv * (dp[nt][e] - ((e >> 1) ? d1 : d0));
        }
      uint32_t dsf[4][4];
      pack_p(dsf, s);
      pv_block<HD>(dq, dsf, sK, kb, lane);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = q0 + g + r * 8;
      if (q < S) {
        bf16* row = dbase + (size_t)q * lddq;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
          if (nt * 8 + 2 * t4 < hd) *reinterpret_cast<uint32_t*>(row + nt * 8 + 2 * t4) = pack_bf162(dq[nt][2 * r] * scale, dq[nt][2 * r + 1] * scale);
      }
    }
  }

  // ---- pass B: this warp owns 16 key rows -> dV = P^T dO,  dK = scale * dS^T Q   (all tiles transposed: rows = keys, cols = queries)
  for (int slab = warp; slab * 16 < S; slab += 8) {
    const int t0 = slab * 16;
    uint32_t kf[KS][4], vf[KS][4];
    load_afrag<HD>(kf, sK, t0, lane);
    load_afrag<HD>(vf, sV, t0, lane);
    float dk[NT][4], dv[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) { dk[nt][e] = 0.f; dv[nt][e] = 0.f; }
    for (int qb = 0; qb < Sp; qb += 64) {
      float s[8][4], dp[8][4];
      qk_block<HD>(s, kf, sQ, qb, lane);    // S^T[t, q]
      qk_block<HD>(dp, vf, sDO, qb, lane);  // dP^T[t, q]
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int q = qb + nt * 8 + 2 * t4 + (e & 1);
          const int t = t0 + g + (e >> 1) * 8;
          float v = s[nt][e] * sc2;
          if (masked || t >= S) v += mask_term(amask, kpm, b, S, q, t);
          const float pv = exp2f(v - sLse[q]);  // padded queries: lse = +inf -> 0
          s[nt][e] = pv;
          dp[nt][e] = pv * (dp[nt][e] - sD[q]);
        }
      uint32_t pf[4][4];
      pack_p(pf, s);
      pv_block<HD>(dv, pf, sDO, qb, lane);
      pack_p(pf, dp);
      pv_block<HD>(dk, pf, sQ, qb, lane);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int t = t0 + g + r * 8;
      if (t < S) {
        bf16* row = dbase + (size_t)t * lddq;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          if (nt * 8 + 2 * t4 >= hd) continue;
          *reinterpret_cast<uint32_t*>(row + C + nt * 8 + 2 * t4) = pack_bf162(dk[nt][2 * r] * scale, dk[nt][2 * r + 1] * scale);
          *reinterpret_cast<uint32_t*>(row + 2 * C + nt * 8 + 2 * t4) = pack_bf162(dv[nt][2 * r], dv[nt][2 * r + 1]);
        }
      }
    }
  }
}

template <int HD>
int launch_fwd(const void* QKV, int ldq, int B, int S, int H, float scale, const float* amask, const uint8_t* kpm, void* O, int ldo, float* LSE,
               cudaStream_t st, int hd) {
  const int Sp = (S + 63) / 64 * 64;
  const size_t smem = (size_t)3 * Sp * MhaCfg<HD>::LD * 2;
  static bool attr = false;
  if (!attr) { CVB_CUDA(cudaFuncSetAttribute(mha_fwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  CVB_CUDA(cvb_launch(mha_fwd_kernel<HD>, B * H, 128, smem, st, static_cast<const bf16*>(QKV), ldq, S, H, scale, amask, kpm, static_cast<bf16*>(O), ldo, LSE, hd));
  CVB_LAUNCH_CHECK();
  return 0;
}
template <int HD>
int launch_bwd(const void* QKV, int ldq, const void* O, const void* DO, int ldo, const float* LSE, int B, int S, int H, float scale,
               const float* amask, const uint8_t* kpm, void* DQKV, int lddq, cudaStream_t st, int hd) {
  const int Sp = (S + 63) / 64 * 64;
  const size_t smem = (size_t)4 * Sp * MhaCfg<HD>::LD * 2 + (size_t)2 * Sp * 4;
  static bool attr = false;
  if (!attr) { CVB_CUDA(cudaFuncSetAttribute(mha_bwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  CVB_CUDA(cvb_launch(mha_bwd_kernel<HD>, B * H, 256, smem, st, static_cast<const bf16*>(QKV), ldq, static_cast<const bf16*>(O),
                      static_cast<const bf16*>(DO), ldo, LSE, S, H, scale, amask, kpm, static_cast<bf16*>(DQKV), lddq, hd));
  CVB_LAUNCH_CHECK();
  return 0;
}

int check_common(const char* who, const void* QKV, int ldq, int B, int S, int H, int head_dim, int ldo) {
  CVB_CHECK(QKV && B > 0 && S > 0 && H > 0, "%s: bad arguments", who);
  CVB_CHECK(head_dim >= 2 && head_dim <= 64 && head_dim % 2 == 0, "%s: head_dim %d not supported (even values up to 64)", who, head_dim);
  CVB_CHECK(S <= 256 || head_dim == 64, "%s: sequence length %d > 256 needs head_dim 64 (got %d): the streaming kernels are head_dim-64 only, the "
            "other head dims keep K/V of one head in shared memory", who, S, head_dim);
  CVB_CHECK(ldq % 8 == 0 && ldo % 8 == 0 && ldq >= 3 * H * head_dim && ldo >= H * head_dim && cvb_aligned16(QKV), "%s: bad leading dimensions / alignment", who);
  return 0;
}

// Which kernels serve a head.  Forward and backward ask the same question, so they always agree (the backward reads the forward's LSE).
//   head_dim != 64                          mma.sync (this file; S <= 256, enforced by check_common)
//   head_dim 64, S > 256                    streaming wgmma (mha_long.cu), with or without masks
//   head_dim 64, S <= 256, additive mask    mma.sync: it reads the [S, S] mask in coalesced tiles, where the wgmma score fragments would
//                                           gather single values (the causal CLIP text tower, S = 77)
//   head_dim 64, S <= 256, otherwise        register-resident wgmma (mha_tc.cu)
// g_mode (cvb_set_mha_impl, cross-checks only) overrides the choice where another family can run the shape.
enum class MhaPath { Mma, Tc, Long };
int g_mode = 0;  // 0 automatic, 1 mma.sync wherever it runs, 2 streaming for every head_dim-64 shape

MhaPath route(int S, int head_dim, bool additive_mask) {
  if (head_dim != 64) return MhaPath::Mma;
  if (S > 256 || g_mode == 2) return MhaPath::Long;
  if (additive_mask || g_mode == 1) return MhaPath::Mma;
  return MhaPath::Tc;
}

}  // namespace

// head_dim 64 launchers: register-resident wgmma (mha_tc.cu: S <= 256, key-padding mask only) and streaming wgmma (mha_long.cu: any S)
int cvb_mha_fwd_tc(const void* QKV, int ldq, int B, int S, int H, float scale, const unsigned char* kpm, void* O, int ldo, float* LSE, cudaStream_t st);
int cvb_mha_bwd_tc(const void* QKV, int ldq, const void* O, const void* DO, int ldo, const float* LSE, int B, int S, int H, float scale,
                   const unsigned char* kpm, void* DQKV, int lddq, cudaStream_t st);
int cvb_mha_fwd_long(const void* QKV, int ldq, int B, int S, int H, float scale, const float* amask, const unsigned char* kpm, void* O, int ldo,
                     float* LSE, cudaStream_t st);
int cvb_mha_bwd_long(const void* QKV, int ldq, const void* O, const void* DO, int ldo, const float* LSE, int B, int S, int H, float scale,
                     const float* amask, const unsigned char* kpm, void* DQKV, int lddq, cudaStream_t st);

extern "C" int cvb_set_mha_impl(int mode) {
  const int old = g_mode;
  g_mode = (mode == 1 || mode == 2) ? mode : 0;
  return old;
}

extern "C" int cvb_mha_fwd(const void* QKV, int ldq, int B, int S, int H, int head_dim, float scale, const float* attn_mask,
                           const unsigned char* key_padding_mask, void* O, int ldo, float* LSE, cvb_stream_t stream) {
  if (check_common("cvb_mha_fwd", QKV, ldq, B, S, H, head_dim, ldo)) return 1;
  CVB_CHECK(O && LSE && cvb_aligned16(O), "cvb_mha_fwd: null / misaligned output");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const MhaPath path = route(S, head_dim, attn_mask != nullptr);
  if (path == MhaPath::Long) return cvb_mha_fwd_long(QKV, ldq, B, S, H, scale, attn_mask, key_padding_mask, O, ldo, LSE, st);
  if (path == MhaPath::Tc) return cvb_mha_fwd_tc(QKV, ldq, B, S, H, scale, key_padding_mask, O, ldo, LSE, st);
  if (head_dim <= 16) return launch_fwd<16>(QKV, ldq, B, S, H, scale, attn_mask, key_padding_mask, O, ldo, LSE, st, head_dim);
  if (head_dim <= 32) return launch_fwd<32>(QKV, ldq, B, S, H, scale, attn_mask, key_padding_mask, O, ldo, LSE, st, head_dim);
  return launch_fwd<64>(QKV, ldq, B, S, H, scale, attn_mask, key_padding_mask, O, ldo, LSE, st, head_dim);
}

extern "C" int cvb_mha_bwd(const void* QKV, int ldq, const void* O, const void* DO, int ldo, const float* LSE, int B, int S, int H, int head_dim,
                           float scale, const float* attn_mask, const unsigned char* key_padding_mask, void* DQKV, int lddq, cvb_stream_t stream) {
  if (check_common("cvb_mha_bwd", QKV, ldq, B, S, H, head_dim, ldo)) return 1;
  CVB_CHECK(O && DO && LSE && DQKV && cvb_aligned16(O) && cvb_aligned16(DO) && cvb_aligned16(DQKV) && lddq % 8 == 0 && lddq >= 3 * H * head_dim,
            "cvb_mha_bwd: null / misaligned operand");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const MhaPath path = route(S, head_dim, attn_mask != nullptr);
  if (path == MhaPath::Long) return cvb_mha_bwd_long(QKV, ldq, O, DO, ldo, LSE, B, S, H, scale, attn_mask, key_padding_mask, DQKV, lddq, st);
  if (path == MhaPath::Tc) return cvb_mha_bwd_tc(QKV, ldq, O, DO, ldo, LSE, B, S, H, scale, key_padding_mask, DQKV, lddq, st);
  if (head_dim <= 16) return launch_bwd<16>(QKV, ldq, O, DO, ldo, LSE, B, S, H, scale, attn_mask, key_padding_mask, DQKV, lddq, st, head_dim);
  if (head_dim <= 32) return launch_bwd<32>(QKV, ldq, O, DO, ldo, LSE, B, S, H, scale, attn_mask, key_padding_mask, DQKV, lddq, st, head_dim);
  return launch_bwd<64>(QKV, ldq, O, DO, ldo, LSE, B, S, H, scale, attn_mask, key_padding_mask, DQKV, lddq, st, head_dim);
}
