// Shared device/host helpers for libcvnets_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/cvnets_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libcvnets_b200 targets sm_90a (H100) only"
#endif

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

// ---------------------------------------------------------------------------------------------- error handling
void cvb_set_error(const char* fmt, ...);
#define CVB_CHECK(cond, ...)            \
  do {                                  \
    if (!(cond)) {                      \
      cvb_set_error(__VA_ARGS__);       \
      return 1;                         \
    }                                   \
  } while (0)
// variadic: the call's template argument lists may hold commas
#define CVB_CUDA(...)                                                                    \
  do {                                                                                   \
    cudaError_t e_ = (__VA_ARGS__);                                                      \
    if (e_ != cudaSuccess) {                                                             \
      (void)cudaGetLastError(); /* reported here: do not leave it for the next caller */ \
      cvb_set_error("%s:%d CUDA error: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); \
      return 2;                                                                          \
    }                                                                                    \
  } while (0)

static inline bool cvb_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
int cvb_num_sms();
// Order-independent gradient accumulation.  Partial sums that many CTAs (or warps) contribute are added in fp64: the few fp32 addends of
// one element sum exactly there, so the result does not depend on the order in which they arrive and two runs of a step are bitwise equal.
// DetScratch holds that fp64 scratch, stream-ordered (capturable).  alloc: n zeroed elements; add: dst[r * ld + c] += scratch[offset +
// r * cols + c]; release: free it after the adds.  An early return frees it in the destructor and keeps the first failure's message.
class DetScratch {
 public:
  explicit DetScratch(cudaStream_t st) : st_(st) {}
  DetScratch(const DetScratch&) = delete;
  DetScratch& operator=(const DetScratch&) = delete;
  ~DetScratch();
  int alloc(size_t n);
  int add(size_t offset, float* dst, int rows, int cols, int ld);
  int release();
  double* data() const { return p_; }

 private:
  cudaStream_t st_;
  double* p_ = nullptr;
};

// ---------------------------------------------------------------------------------------------- small device helpers
// SiLU through ONE special-function op: sigmoid(z) = 0.5 + 0.5 tanh(z/2) with tanh.approx.f32 (MUFU.TANH, max abs error 2^-11), instead of
// ex2 + rcp (two MUFU ops at 16 / clk / SM: the SiLU of a large activation tensor would be bound by the MUFU pipe).  The
// absolute error of silu is <= |z| * 2.5e-4 -- below bf16 resolution of every value that is not itself negligible.
__device__ __forceinline__ float tanh_approx_f(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigmoid_f(float z) { return fmaf(0.5f, tanh_approx_f(0.5f * z), 0.5f); }
__device__ __forceinline__ float silu_f(float z) {
  const float h = 0.5f * z;
  return fmaf(h, tanh_approx_f(h), h);
}
// d/dz [z*sigmoid(z)] = s*(1 + z*(1-s))
__device__ __forceinline__ float silu_grad_f(float z) {
  const float s = sigmoid_f(z);
  return s * (1.0f + z * (1.0f - s));
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__device__ __forceinline__ uint32_t pack_bf162(float lo, float hi) {
  bf162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf162(uint32_t u) {
  bf162 v = *reinterpret_cast<bf162*>(&u);
  return __bfloat1622float2(v);
}
// fp32 arithmetic on a register pair.  Hopper has no packed f32x2 instructions: these are two scalar ops each, with the same
// round-to-nearest results (fma stays fused), so callers written for pairs keep their numerics.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
// 8 bf16 <-> 8 floats
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  float2 a = unpack_bf162(u.x), b = unpack_bf162(u.y), c = unpack_bf162(u.z), d = unpack_bf162(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 u;
  u.x = pack_bf162(f[0], f[1]); u.y = pack_bf162(f[2], f[3]); u.z = pack_bf162(f[4], f[5]); u.w = pack_bf162(f[6], f[7]);
  return u;
}
__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
// streaming (read-once / write-once) 16-byte accesses: do not pollute L1
__device__ __forceinline__ uint4 ldg16_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void stg16(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// cp.async 16B with zero-fill when !pred (src-size 0)
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr, bool pred) {
  int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_addr), "l"(gptr), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
__device__ __forceinline__ void mma_bf16_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// apply a per-channel "load mode" to one value
__device__ __forceinline__ float apply_mode(int mode, float x, float p0, float p1) {
  switch (mode) {
    case CVB_A_AFF: return fmaf(p0, x, p1);
    case CVB_A_AFF_SILU: return silu_f(fmaf(p0, x, p1));
    case CVB_A_SILU: return silu_f(x);
    default: return x;
  }
}

// ---------------------------------------------------------------------------------------------- programmatic dependent launch
// Every kernel of the library is launched with the programmatic-stream-serialization attribute: its CTAs may become resident
// while the previous kernel in the stream is still draining, run their private set-up (mbarrier init,
// tensor-map prefetch), and block in pdl_wait() until the previous grid has completed and flushed its memory.  RULES: nothing
// produced by an earlier kernel is read, and no global memory is written, before pdl_wait(); every kernel executes
// pdl_wait() in every thread (so "grid B complete" always implies "grid A complete" along the stream).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
int cvb_pdl_enabled();
// Returns the launch's error, or the error pending after it (cudaGetLastError) when the launch itself succeeded.
template <typename... KArgs, typename... Args>
static inline cudaError_t cvb_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cvb_pdl_enabled() ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  return e != cudaSuccess ? e : cudaGetLastError();
}
// Opts the kernel in to `bytes` of dynamic shared memory (past the default 48 KB) on its first call.  The flag is keyed on the kernel
// itself, so kernels with the same parameter list keep their own.
template <auto Kernel>
static inline cudaError_t cvb_smem_optin(int bytes) {
  static bool done = false;
  if (done) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  done = e == cudaSuccess;
  return e;
}

// ---------------------------------------------------------------------------------------------- TMA + mbarrier (sm_90a)
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint, no -lcuda)

// Host: tensor map of a channels-last bf16 feature map [B, H, W, C] with a [1, boxH, boxW, boxC] box (boxC * 2 bytes <= 128),
// no swizzle, zero fill for out-of-bounds elements (the conv halo).
int cvb_make_tmap_nhwc(CUtensorMap* map, const void* base, int B, int H, int W, int C, int boxH, int boxW, int boxC);
// Host: tensor map of a row-major bf16 matrix [rows, cols] (leading dimension ld elements) with a [box_rows, box_cols] box.  The swizzle
// follows from the box width:
//   32 columns: 64-byte swizzle; the shared-memory image is exactly the 64-byte-row XOR layout (swz64) the GEMM's ldmatrix addressing uses.
//   64 columns: 128-byte swizzle; the image is the canonical MN-major SWIZZLE_128B wgmma operand layout (8-row x 128-byte atoms) when the
//               ROWS are the reduction dimension (weight-gradient GEMM).
int cvb_make_tmap_2d(CUtensorMap* map, const void* base, int64_t rows, int cols, int ld, int box_rows, int box_cols);

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// make generic-proxy writes/reads of smem visible to the async proxy (TMA) before it overwrites the buffer
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
// 2-D tiled TMA load: coordinates (col, row)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int col, int row) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(col), "r"(row)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }

// ---------------------------------------------------------------------------------------------- wgmma (sm_90a warpgroup MMA)
// Shared-memory matrix descriptor: start address, leading / stride byte offsets (16-byte units), layout type in bits [62,64)
// (1 = 128-byte swizzle, 2 = 64-byte swizzle).  K-major swizzled operands ignore the leading offset; MN-major SWIZZLE_128B
// operands use it as the distance between 64-element groups of the M/N dimension and the stride offset between 8-row k groups.
enum { WG_SW128 = 1, WG_SW64 = 2 };
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, int layout) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the accumulator registers live and ordered around the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_reg_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 operands from shared memory, fp32 accumulator in registers (N / 2 per thread).
// TA / TB: operand is MN-major (transposed) instead of K-major.  Accumulator fragment: thread t of the warpgroup holds, for every
// 8-column block j, rows 16 (t / 32) + (t % 32) / 4 (+ 8 for the odd pair) and columns 8 j + 2 (t % 4) + {0, 1}.
#define CVB_WG_R8(b) "+f"(d[b + 0]), "+f"(d[b + 1]), "+f"(d[b + 2]), "+f"(d[b + 3]), "+f"(d[b + 4]), "+f"(d[b + 5]), "+f"(d[b + 6]), "+f"(d[b + 7])
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1, %35, %36;\n\t}"
      : CVB_WG_R8(0), CVB_WG_R8(8), CVB_WG_R8(16), CVB_WG_R8(24)
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}"
      : CVB_WG_R8(0), CVB_WG_R8(8), CVB_WG_R8(16), CVB_WG_R8(24), CVB_WG_R8(32), CVB_WG_R8(40), CVB_WG_R8(48), CVB_WG_R8(56)
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
// Same with A [64 x 16] from registers: a[0..3] = bf16 pairs (row g, cols 2t..), (g + 8, 2t..), (g, 2t + 8..), (g + 8, 2t + 8..) of warp w's
// 16 rows, g = lane / 4, t = lane % 4 -- i.e. accumulator columns 16 kk .. 16 kk + 15 of an m64nN result, packed, feed k-step kk directly.
template <int TB>
__device__ __forceinline__ void wgmma_m64n64_rs(float* d, const uint32_t* a, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32,%33,%34,%35}, %36, p, 1, 1, %38;\n\t}"
      : CVB_WG_R8(0), CVB_WG_R8(8), CVB_WG_R8(16), CVB_WG_R8(24)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate), "n"(TB));
}
#undef CVB_WG_R8

// 4-D tiled TMA load: coordinates innermost first (c, w, h, b); completes `bytes of the box` on the mbarrier
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c, int w, int h, int b) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(b)
               : "memory");
}
