// Streaming (flash-style) wgmma attention for head_dim == 64 and any sequence length, sm_90a.  Same contract as mha.cu / mha_tc.cu.
//
// mha_tc.cu keeps a whole head in shared memory and whole score rows in registers, which caps S at 256.  Here K / V (forward) and
// Q / dO (backward) stream through a 3-stage shared-memory ring in 64-row tiles, so nothing on chip grows with S (ViT / CLIP at the
// multi-scale recipes' 256-320 px crops: S = 257 .. 401; 384 px fine-tuning: S = 577; 512 px: S = 1025).  The router in mha.cu sends
// every head_dim-64 head with S > 256 here, with or without masks; test mode 2 of cvb_set_mha_impl sends the shorter ones too.
//
// Operand images are the ones mha_tc.cu uses, from the same helpers (mha_wgmma.cuh): one [64 rows x 64 ch] SWIZZLE_128B TMA box per
// tile, read as the K-major operand (rows = M / N) or as the MN-major operand (rows = K) of a wgmma; P and dS go from the accumulator
// registers straight into the A operand of the next wgmma.  Warp 8 of every CTA is the TMA producer (full / empty mbarrier pair per stage); warps 0-7 are two consumer
// warpgroups of 64 rows each.
//
// Forward, one CTA per (sample, head, 128 queries): online softmax in the exp2 domain (running row max and sum, O rescaled per key tile).
// O bf16, LSE = m + log2 l exactly as mha_tc_fwd_kernel (scaled-score exp2 domain), so the backward of either family reads it.
//
// Backward, bitwise reproducible (no atomics; every output element is written by exactly one thread):
//   mha_long_d_kernel     D[b, h, q] = sum_c dO O (fp32), once
//   mha_long_dkv_kernel   one CTA per (sample, head, 128 keys): streams Q / dO tiles, P^T and dS^T from LSE and D, dV += P^T dO, dK += dS^T Q
//   mha_long_dq_kernel    one CTA per (sample, head, 128 queries): streams K / V tiles, recomputes P and dS, dQ += dS K
// The price of determinism is the recompute of Q K^T and dO V^T in the dQ kernel: 7 instead of 5 m64n64 products per (64 x 64) block.
#include "mha_wgmma.cuh"

namespace {

constexpr int NST = 3;           // ring stages
constexpr int THREADS = 288;     // two consumer warpgroups + one producer warp
constexpr int PRODUCER = 256;    // first thread of the producer warp

// Shared layout of every kernel: two own [128 rows] operand images (Q, or K | V, or Q | dO: 4 boxes), then NST stages of two streamed boxes.
struct Smem {
  uint8_t* own;    // 4 boxes: own operand 0 rows 0-63, 64-127, own operand 1 rows 0-63, 64-127
  uint8_t* ring;   // NST x 2 boxes
};
constexpr size_t SMEM_BYTES = (size_t)(4 + 2 * NST) * BOX64 + 1024;

__device__ __forceinline__ Smem carve(uint8_t* raw) {
  uint8_t* p = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  return Smem{p, p + 4 * BOX64};
}

// Producer: stream tiles j = 0 .. ntiles-1 (rows row0 + 64 j) of two column blocks (c0, c1) of two tensor maps into the ring.
__device__ __forceinline__ void produce(const CUtensorMap* m0, int c0, const CUtensorMap* m1, int c1, int row0, int ntiles, uint8_t* ring, uint64_t* full,
                                        uint64_t* empty) {
  for (int j = 0; j < ntiles; ++j) {
    const int s = j % NST;
    if (j >= NST) mbar_wait(&empty[s], ((j / NST) & 1) ^ 1);  // consumers released the stage's previous use (tile j - NST)
    mbar_expect_tx(&full[s], 2 * BOX64);
    tma_load_2d(ring + (2 * s) * BOX64, m0, &full[s], c0, row0 + 64 * j);
    tma_load_2d(ring + (2 * s + 1) * BOX64, m1, &full[s], c1, row0 + 64 * j);
  }
}

// Common prologue: barrier init, own operands (two 128-row blocks: map m0 column c0, map m1 column c1; m1 == nullptr: only m0, 2 boxes).
__device__ __forceinline__ void prologue(uint64_t* bar_own, uint64_t* full, uint64_t* empty, const CUtensorMap* m0, int c0, const CUtensorMap* m1, int c1,
                                         int row0, uint8_t* own) {
  const int tid = threadIdx.x;
  if (tid == PRODUCER) {
    mbar_init(bar_own, 1);
    for (int s = 0; s < NST; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  if (tid == PRODUCER) {
    mbar_expect_tx(bar_own, (m1 ? 4 : 2) * BOX64);
    tma_load_2d(own, m0, bar_own, c0, row0);
    tma_load_2d(own + BOX64, m0, bar_own, c0, row0 + 64);
    if (m1) {
      tma_load_2d(own + 2 * BOX64, m1, bar_own, c1, row0);
      tma_load_2d(own + 3 * BOX64, m1, bar_own, c1, row0 + 64);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------- forward
__global__ void __launch_bounds__(THREADS, 1)
    mha_long_fwd_kernel(const __grid_constant__ CUtensorMap tm, int S, int H, int NQT, float scale, const float* __restrict__ amask,
                        const uint8_t* __restrict__ kpm, bf16* __restrict__ O, int ldo, float* __restrict__ LSE) {
  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7;
  int bid = blockIdx.x;
  const int qt = bid % NQT;
  bid /= NQT;
  const int h = bid % H, b = bid / H;
  const int C = H * 64, NKT = (S + 63) / 64;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const Smem sm = carve(smem_raw);
  __shared__ __align__(8) uint64_t bar_q, full[NST], empty[NST];
  prologue(&bar_q, full, empty, &tm, h * 64, nullptr, 0, b * S + qt * 128, sm.own);
  if (tid >= PRODUCER) {
    if (tid == PRODUCER) produce(&tm, C + h * 64, &tm, 2 * C + h * 64, b * S, NKT, sm.ring, full, empty);
    return;
  }

  const int rl = ((tid & 127) >> 5) * 16 + (lane >> 2);  // query row (within the warpgroup's 64) of acc[4j + {0,1}]; + 8 for {2,3}
  const int q0 = qt * 128 + wg * 64;
  const float sc2 = scale * LOG2E;
  const bool masked = (amask != nullptr) || (kpm != nullptr);
  const uint32_t aQ = smem_u32(sm.own) + wg * BOX64, aRing = smem_u32(sm.ring);

  float o[32], m[2] = {-CUDART_INF_F, -CUDART_INF_F}, l[2] = {0.f, 0.f};  // l: this thread's partial row sums
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait(&bar_q, 0);
  for (int j = 0; j < NKT; ++j) {
    const int s = j % NST;
    const uint32_t aK = aRing + (2 * s) * BOX64, aV = aK + BOX64;
    mbar_wait(&full[s], (j / NST) & 1);
    float sacc[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(sacc, desc_k(aQ + k * 32), desc_k(aK + k * 32), k ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<32>(sacc);
    float mt[2] = {m[0], m[1]};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hh = (i >> 1) & 1, q = q0 + rl + 8 * hh, t = j * 64 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      float v = -CUDART_INF_F;
      if (t < S) {
        v = sacc[i] * sc2;
        if (masked) v += mask_add(amask, kpm, b, S, q, t);
      }
      sacc[i] = v;
      mt[hh] = fmaxf(mt[hh], v);
    }
    float alpha[2], msafe[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mt[hh] = fmaxf(mt[hh], __shfl_xor_sync(0xffffffffu, mt[hh], 1));
      mt[hh] = fmaxf(mt[hh], __shfl_xor_sync(0xffffffffu, mt[hh], 2));
      msafe[hh] = (mt[hh] == -CUDART_INF_F) ? 0.f : mt[hh];  // a row masked so far must not produce inf - inf
      alpha[hh] = ex2(m[hh] - msafe[hh]);                     // 0 on the first tile (m = -inf)
      m[hh] = mt[hh];
      l[hh] *= alpha[hh];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hh = (i >> 1) & 1;
      const float pv = ex2(sacc[i] - msafe[hh]);
      sacc[i] = pv;
      l[hh] += pv;
      o[i] *= alpha[hh];
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t a[4];
      to_a_frag(sacc, kk, a);
      wgmma_m64n64_rs<1>(o, a, desc_mn(aV + kk * 16 * 128), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<32>(o);
    if (lane == 0) mbar_arrive(&empty[s]);  // this warp's reads of the stage are complete
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
  }
  // a fully masked row gives 0 * inf = NaN, like softmax over an all -inf row in the reference
  const float inv[2] = {1.0f / l[0], 1.0f / l[1]};
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] *= inv[(i >> 1) & 1];
  store_acc(O + (size_t)b * S * ldo + h * 64, ldo, o, 1.0f, q0, S);
  if ((lane & 3) == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int q = q0 + rl + 8 * hh;
      if (q < S) LSE[((size_t)b * H + h) * S + q] = m[hh] + log2f(l[hh]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------ backward
// D[b, h, q] = sum_c dO[b, q, h, c] O[b, q, h, c], one thread per (b, q, h)
__global__ void __launch_bounds__(256) mha_long_d_kernel(const bf16* __restrict__ O, const bf16* __restrict__ DO, int ldo, int B, int S, int H,
                                                          float* __restrict__ D) {
  pdl_wait();
  pdl_trigger();
  const int64_t total = (int64_t)B * S * H;
  for (int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * 256) {
    const int h = (int)(idx % H);
    const int64_t row = idx / H;  // b * S + q
    const bf16* orow = O + row * ldo + h * 64;
    const bf16* drow = DO + row * ldo + h * 64;
    float d = 0.f;
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
      float a[8], c[8];
      unpack8(ldg16(orow + ch * 8), a);
      unpack8(ldg16(drow + ch * 8), c);
#pragma unroll
      for (int e = 0; e < 8; ++e) d = fmaf(a[e], c[e], d);
    }
    const int64_t b = row / S, q = row % S;
    D[(b * H + h) * S + q] = d;
  }
}

// dK, dV of 128 keys: S^T = K Q^T, dP^T = V dO^T per streamed (Q, dO) tile of 64 queries; P^T = exp2(S^T sc2 + mask - LSE), dS^T = P^T (dP^T - D)
__global__ void __launch_bounds__(THREADS, 1)
    mha_long_dkv_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO, const float* __restrict__ LSE,
                        const float* __restrict__ Dv, int S, int H, int NKT, float scale, const float* __restrict__ amask, const uint8_t* __restrict__ kpm,
                        bf16* __restrict__ DQKV, int lddq) {
  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7;
  int bid = blockIdx.x;
  const int kt = bid % NKT;
  bid /= NKT;
  const int h = bid % H, b = bid / H;
  const int C = H * 64, NQB = (S + 63) / 64;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const Smem sm = carve(smem_raw);
  __shared__ __align__(8) uint64_t bar_kv, full[NST], empty[NST];
  prologue(&bar_kv, full, empty, &tmQKV, C + h * 64, &tmQKV, 2 * C + h * 64, b * S + kt * 128, sm.own);
  if (tid >= PRODUCER) {
    if (tid == PRODUCER) produce(&tmQKV, h * 64, &tmDO, h * 64, b * S, NQB, sm.ring, full, empty);
    return;
  }

  const int rl = ((tid & 127) >> 5) * 16 + (lane >> 2);  // key row (within the warpgroup's 64) of acc[4j + {0,1}]; + 8 for {2,3}
  const int k0 = kt * 128 + wg * 64;
  const float sc2 = scale * LOG2E;
  const bool masked = (amask != nullptr) || (kpm != nullptr);
  const uint32_t aK = smem_u32(sm.own) + wg * BOX64, aV = aK + 2 * BOX64, aRing = smem_u32(sm.ring);
  const float* lse = LSE + ((size_t)b * H + h) * S;
  const float* dvec = Dv + ((size_t)b * H + h) * S;

  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait(&bar_kv, 0);
  for (int j = 0; j < NQB; ++j) {
    const int s = j % NST;
    const uint32_t aQ = aRing + (2 * s) * BOX64, aDO = aQ + BOX64;
    mbar_wait(&full[s], (j / NST) & 1);
    float st[32], dpt[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(st, desc_k(aK + k * 32), desc_k(aQ + k * 32), k ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(dpt, desc_k(aV + k * 32), desc_k(aDO + k * 32), k ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<32>(st);
    wgmma_reg_fence<32>(dpt);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int t = k0 + rl + 8 * ((i >> 1) & 1), q = j * 64 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      float pv = 0.f, ds = 0.f;
      if (q < S && t < S) {  // per-query LSE / D of the score column: global, L2-resident
        float v = fmaf(st[i], sc2, -__ldg(lse + q));
        if (masked) v += mask_add(amask, kpm, b, S, q, t);
        pv = ex2(v);
        ds = pv * (dpt[i] - __ldg(dvec + q));
        if (pv == 0.f) ds = 0.f;  // masked keys: exactly zero whatever dP holds
      }
      st[i] = pv;
      dpt[i] = ds;
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // reduction over the 64 queries of the tile
      uint32_t a[4];
      to_a_frag(st, kk, a);
      wgmma_m64n64_rs<1>(dv, a, desc_mn(aDO + kk * 16 * 128), 1u);
      to_a_frag(dpt, kk, a);
      wgmma_m64n64_rs<1>(dk, a, desc_mn(aQ + kk * 16 * 128), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<32>(dv);
    wgmma_reg_fence<32>(dk);
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  bf16* dbase = DQKV + (size_t)b * S * lddq + h * 64;
  store_acc(dbase + C, lddq, dk, scale, k0, S);
  store_acc(dbase + 2 * C, lddq, dv, 1.0f, k0, S);
}

// dQ of 128 queries: S = Q K^T, dP = dO V^T per streamed (K, V) tile of 64 keys; P = exp2(S sc2 + mask - LSE), dS = P (dP - D), dQ += dS K
__global__ void __launch_bounds__(THREADS, 1)
    mha_long_dq_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO, const float* __restrict__ LSE,
                       const float* __restrict__ Dv, int S, int H, int NQT, float scale, const float* __restrict__ amask, const uint8_t* __restrict__ kpm,
                       bf16* __restrict__ DQKV, int lddq) {
  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7;
  int bid = blockIdx.x;
  const int qt = bid % NQT;
  bid /= NQT;
  const int h = bid % H, b = bid / H;
  const int C = H * 64, NKB = (S + 63) / 64;

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const Smem sm = carve(smem_raw);
  __shared__ __align__(8) uint64_t bar_q, full[NST], empty[NST];
  prologue(&bar_q, full, empty, &tmQKV, h * 64, &tmDO, h * 64, b * S + qt * 128, sm.own);
  if (tid >= PRODUCER) {
    if (tid == PRODUCER) produce(&tmQKV, C + h * 64, &tmQKV, 2 * C + h * 64, b * S, NKB, sm.ring, full, empty);
    return;
  }

  const int rl = ((tid & 127) >> 5) * 16 + (lane >> 2);  // query row (within the warpgroup's 64) of acc[4j + {0,1}]; + 8 for {2,3}
  const int q0 = qt * 128 + wg * 64;
  const float sc2 = scale * LOG2E;
  const bool masked = (amask != nullptr) || (kpm != nullptr);
  const uint32_t aQ = smem_u32(sm.own) + wg * BOX64, aDO = aQ + 2 * BOX64, aRing = smem_u32(sm.ring);
  float lq[2], dq2[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = q0 + rl + 8 * hh;
    lq[hh] = q < S ? LSE[((size_t)b * H + h) * S + q] : 0.f;
    dq2[hh] = q < S ? Dv[((size_t)b * H + h) * S + q] : 0.f;
  }

  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  mbar_wait(&bar_q, 0);
  for (int j = 0; j < NKB; ++j) {
    const int s = j % NST;
    const uint32_t aK = aRing + (2 * s) * BOX64, aV = aK + BOX64;
    mbar_wait(&full[s], (j / NST) & 1);
    float sa[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(sa, desc_k(aQ + k * 32), desc_k(aK + k * 32), k ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n64<0, 0>(dp, desc_k(aDO + k * 32), desc_k(aV + k * 32), k ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<32>(sa);
    wgmma_reg_fence<32>(dp);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hh = (i >> 1) & 1;
      const int q = q0 + rl + 8 * hh, t = j * 64 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      float ds = 0.f;
      if (q < S && t < S) {
        float v = fmaf(sa[i], sc2, -lq[hh]);
        if (masked) v += mask_add(amask, kpm, b, S, q, t);
        const float pv = ex2(v);
        ds = pv * (dp[i] - dq2[hh]);
        if (pv == 0.f) ds = 0.f;
      }
      sa[i] = ds;
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // reduction over the 64 keys of the tile
      uint32_t a[4];
      to_a_frag(sa, kk, a);
      wgmma_m64n64_rs<1>(dq, a, desc_mn(aK + kk * 16 * 128), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<32>(dq);
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  store_acc(DQKV + (size_t)b * S * lddq + h * 64, lddq, dq, scale, q0, S);
}

}  // namespace

int cvb_mha_fwd_long(const void* QKV, int ldq, int B, int S, int H, float scale, const float* amask, const unsigned char* kpm, void* O, int ldo,
                     float* LSE, cudaStream_t st) {
  const int NQT = (S + 127) / 128;
  CUtensorMap tm;
  if (cvb_make_tmap_2d(&tm, QKV, (int64_t)B * S, 3 * H * 64, ldq, 64, 64)) return 1;
  CVB_CUDA(cvb_smem_optin<mha_long_fwd_kernel>((int)SMEM_BYTES));
  CVB_CUDA(cvb_launch(mha_long_fwd_kernel, B * H * NQT, THREADS, SMEM_BYTES, st, tm, S, H, NQT, scale, amask, kpm, static_cast<bf16*>(O), ldo, LSE));
  return 0;
}

int cvb_mha_bwd_long(const void* QKV, int ldq, const void* O, const void* DO, int ldo, const float* LSE, int B, int S, int H, float scale,
                     const float* amask, const unsigned char* kpm, void* DQKV, int lddq, cudaStream_t st) {
  const int NT = (S + 127) / 128;
  CUtensorMap tmQKV, tmDO;
  if (cvb_make_tmap_2d(&tmQKV, QKV, (int64_t)B * S, 3 * H * 64, ldq, 64, 64)) return 1;
  if (cvb_make_tmap_2d(&tmDO, DO, (int64_t)B * S, H * 64, ldo, 64, 64)) return 1;
  CVB_CUDA(cvb_smem_optin<mha_long_dkv_kernel>((int)SMEM_BYTES));
  CVB_CUDA(cvb_smem_optin<mha_long_dq_kernel>((int)SMEM_BYTES));
  // D: stream-ordered scratch from the device pool (DetScratch: fp64 elements, zero-filled; used here as B*H*S floats)
  DetScratch ws(st);
  if (ws.alloc(((size_t)B * H * S + 1) / 2)) return 2;
  float* Dv = reinterpret_cast<float*>(ws.data());
  const int64_t rows = (int64_t)B * S * H;
  int64_t grid = (rows + 255) / 256;
  if (grid > 16 * (int64_t)cvb_num_sms()) grid = 16 * (int64_t)cvb_num_sms();
  CVB_CUDA(cvb_launch(mha_long_d_kernel, (int)grid, 256, 0, st, static_cast<const bf16*>(O), static_cast<const bf16*>(DO), ldo, B, S, H, Dv));
  CVB_CUDA(cvb_launch(mha_long_dkv_kernel, B * H * NT, THREADS, SMEM_BYTES, st, tmQKV, tmDO, LSE, static_cast<const float*>(Dv), S, H, NT, scale, amask,
                      kpm, static_cast<bf16*>(DQKV), lddq));
  CVB_CUDA(cvb_launch(mha_long_dq_kernel, B * H * NT, THREADS, SMEM_BYTES, st, tmQKV, tmDO, LSE, static_cast<const float*>(Dv), S, H, NT, scale, amask,
                      kpm, static_cast<bf16*>(DQKV), lddq));
  return ws.release();
}
