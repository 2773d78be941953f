// Dilated depthwise 3x3 convolution (stride 1, pad = dilation), NHWC bf16, forward and fused backward (sm_90a).
//
// SURVEY.md 8f row 4: segmentation backbones run MobileViTv2 with output_stride 8 / 16, which replaces the stride of layer_4 / layer_5
// by dilation 2 / 4 in their depthwise convs (cvnets/models/classification/base_image_encoder.py:38-47, mobilevit_v2.py:176-191;
// InvertedResidual conv_3x3 at cvnets/modules/mobilenetv2.py:194-207, MobileViTBlockv2 local_rep at mobilevit_block.py:369-379).
// The walk kernels of dwconv.cu keep a dense 3x3 neighbourhood in registers, which a dilated stencil does not have; these layers are the
// late, small feature maps (<= 32x32 at 256x256 input, L2 resident), so this is a direct gather: one thread = one pixel x 8 channels
// (16-byte accesses, a warp covers consecutive channel chunks of consecutive pixels), same load modes, same fused outputs and the same
// rounding points as the walk kernels (cvb_dw_fwd / cvb_dw_bwd dispatch here when args.dilation > 1).
#include "common.cuh"

namespace {

constexpr int DNT = 256;

template <int XMODE>
__device__ __forceinline__ void act8(const uint4& raw, const float* sc, const float* sh, float* a) {
  unpack8(raw, a);
  if (XMODE != CVB_A_RAW) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = fmaf(sc[j], a[j], sh[j]);
      a[j] = (XMODE == CVB_A_AFF_SILU) ? silu_f(z) : z;
    }
  }
}

// block = (chunks of 8 channels handled by threadIdx.x, PY pixel lanes on threadIdx.y); a thread keeps its channel chunk for the whole
// kernel, so weights, parameters and the statistics accumulators live in registers.
template <int XMODE>
__global__ void __launch_bounds__(DNT) dwd_fwd_kernel(const cvb_dw_fwd_args p, int dil, int CC) {
  pdl_wait();
  pdl_trigger();
  __shared__ float s_red[DNT][17];
  const int cx = blockDim.x, py = blockDim.y;
  const int64_t npix = (int64_t)p.B * p.H * p.W;
  float cs[8], cq[8];
  for (int base = 0; base < CC; base += cx) {  // uniform trip count: the block reductions below contain barriers
    const bool live = base + (int)threadIdx.x < CC;
    const int c = (live ? base + (int)threadIdx.x : 0) * 8;
    float w[9][8], sc[8], sh[8];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      *reinterpret_cast<float4*>(w[t]) = __ldg(reinterpret_cast<const float4*>(p.Wt + (size_t)t * p.C + c));
      *reinterpret_cast<float4*>(w[t] + 4) = __ldg(reinterpret_cast<const float4*>(p.Wt + (size_t)t * p.C + c + 4));
    }
    if (XMODE != CVB_A_RAW) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { sc[j] = __ldg(p.x_p0 + c + j); sh[j] = __ldg(p.x_p1 + c + j); }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { cs[j] = 0.f; cq[j] = 0.f; }
    for (int64_t pix = (int64_t)blockIdx.x * py + threadIdx.y; live && pix < npix; pix += (int64_t)gridDim.x * py) {
      const int wq = (int)(pix % p.W), hq = (int)((pix / p.W) % p.H);
      const int64_t img = pix - (int64_t)hq * p.W - wq;  // first pixel of the image
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        const int h = hq + (u - 1) * dil;
        if (h < 0 || h >= p.H) continue;  // zero padding acts on the activated tensor: out-of-image taps contribute nothing
#pragma unroll
        for (int v = 0; v < 3; ++v) {
          const int ww = wq + (v - 1) * dil;
          if (ww < 0 || ww >= p.W) continue;
          const uint4 raw = __ldg(reinterpret_cast<const uint4*>(static_cast<const bf16*>(p.X) + (size_t)(img + (int64_t)h * p.W + ww) * p.C + c));
          float a[8];
          act8<XMODE>(raw, sc, sh, a);
          if (XMODE != CVB_A_RAW) {  // the walk kernels round the activated operand to bf16 when they transform the staged tile
#pragma unroll
            for (int j = 0; j < 8; ++j) a[j] = __bfloat162float(__float2bfloat16(a[j]));
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = fmaf(w[u * 3 + v][j], a[j], acc[j]);
        }
      }
      const uint4 out = pack8(acc);
      *reinterpret_cast<uint4*>(static_cast<bf16*>(p.Y) + (size_t)pix * p.C + c) = out;
      if (p.col_sum) {
        float r[8];
        unpack8(out, r);  // statistics of the stored (rounded) values
#pragma unroll
        for (int j = 0; j < 8; ++j) { cs[j] += r[j]; cq[j] = fmaf(r[j], r[j], cq[j]); }
      }
    }
    if (p.col_sum) {
      // reduce over the pixel lanes of the block, then one fp64 atomic per channel per block
      const int tid = threadIdx.y * cx + threadIdx.x;
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 8; ++j) { s_red[tid][j] = cs[j]; s_red[tid][8 + j] = cq[j]; }
      __syncthreads();
      if (threadIdx.y == 0 && live) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float a = 0.f, b = 0.f;
          for (int y = 0; y < py; ++y) { a += s_red[y * cx + threadIdx.x][j]; b += s_red[y * cx + threadIdx.x][8 + j]; }
          atomicAdd(p.col_sum + c + j, (double)a);
          atomicAdd(p.col_sq + c + j, (double)b);
        }
      }
    }
  }
}

// Backward at INPUT pixel q (stride 1): the neighbourhood dy[q - (t-1)*dil] feeds both products,
//   da[q] = sum_t W[t] * dy[q - (t-1)*dil]          dW[t] += act(x[q]) * dy[q - (t-1)*dil]
// then dX = da * act'(z) (producer's activation backward) and the producer's BN-backward statistics (sum dX, sum dX * x).
template <int GMODE, int XMODE>
__global__ void __launch_bounds__(DNT) dwd_bwd_kernel(const cvb_dw_bwd_args p, int dil, int CC) {
  pdl_wait();
  pdl_trigger();
  __shared__ float s_red[DNT][9];
  const int cx = blockDim.x, py = blockDim.y;
  const int tid = threadIdx.y * cx + threadIdx.x;
  const int64_t npix = (int64_t)p.B * p.H * p.W;
  for (int base = 0; base < CC; base += cx) {  // uniform trip count (barriers in the reductions)
    const bool live = base + (int)threadIdx.x < CC;
    const int c = (live ? base + (int)threadIdx.x : 0) * 8;
    float w[9][8], dw[9][8], sc[8], sh[8], c1[8], c2[8], c3[8], cs[8], cq[8];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      *reinterpret_cast<float4*>(w[t]) = __ldg(reinterpret_cast<const float4*>(p.Wt + (size_t)t * p.C + c));
      *reinterpret_cast<float4*>(w[t] + 4) = __ldg(reinterpret_cast<const float4*>(p.Wt + (size_t)t * p.C + c + 4));
#pragma unroll
      for (int j = 0; j < 8; ++j) dw[t][j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      cs[j] = 0.f; cq[j] = 0.f;
      if (XMODE != CVB_A_RAW) { sc[j] = __ldg(p.x_p0 + c + j); sh[j] = __ldg(p.x_p1 + c + j); }
      if (GMODE == CVB_A_BNB) { c1[j] = __ldg(p.g_p0 + c + j); c2[j] = __ldg(p.g_p1 + c + j); c3[j] = __ldg(p.g_p2 + c + j); }
    }
    for (int64_t pix = (int64_t)blockIdx.x * py + threadIdx.y; live && pix < npix; pix += (int64_t)gridDim.x * py) {
      const int wq = (int)(pix % p.W), hq = (int)((pix / p.W) % p.H);
      const int64_t img = pix - (int64_t)hq * p.W - wq;
      float xr[8], a[8], dact[8], da[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(static_cast<const bf16*>(p.X) + (size_t)pix * p.C + c)), xr);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        da[j] = 0.f;
        if (XMODE == CVB_A_RAW) {
          a[j] = xr[j];
          dact[j] = 1.f;
        } else {
          const float z = fmaf(sc[j], xr[j], sh[j]);
          if (XMODE == CVB_A_AFF_SILU) {
            const float s = sigmoid_f(z);
            a[j] = z * s;
            dact[j] = fmaf(a[j], 1.0f - s, s);
          } else {
            a[j] = z;
            dact[j] = 1.f;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        const int h = hq - (u - 1) * dil;
        if (h < 0 || h >= p.H) continue;
#pragma unroll
        for (int v = 0; v < 3; ++v) {
          const int ww = wq - (v - 1) * dil;
          if (ww < 0 || ww >= p.W) continue;
          const size_t off = (size_t)(img + (int64_t)h * p.W + ww) * p.C + c;
          float dy[8];
          unpack8(__ldg(reinterpret_cast<const uint4*>(static_cast<const bf16*>(p.DZ) + off)), dy);
          if (GMODE == CVB_A_BNB) {
            float y2[8];
            unpack8(__ldg(reinterpret_cast<const uint4*>(static_cast<const bf16*>(p.Y2) + off)), y2);
#pragma unroll
            for (int j = 0; j < 8; ++j) dy[j] = __bfloat162float(__float2bfloat16(fmaf(c1[j], dy[j], fmaf(c2[j], y2[j], c3[j]))));
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            da[j] = fmaf(w[u * 3 + v][j], dy[j], da[j]);
            dw[u * 3 + v][j] = fmaf(a[j], dy[j], dw[u * 3 + v][j]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) da[j] *= dact[j];
      const uint4 out = pack8(da);
      *reinterpret_cast<uint4*>(static_cast<bf16*>(p.DX) + (size_t)pix * p.C + c) = out;
      if (p.col_sum && XMODE != CVB_A_RAW) {
        float r[8];
        unpack8(out, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) { cs[j] += r[j]; cq[j] = fmaf(r[j], xr[j], cq[j]); }
      }
    }
    // ---- block reductions over the pixel lanes: dW (9 taps x 8 channels), then the statistics
#pragma unroll 1
    for (int j = 0; j < 8; ++j) {
      __syncthreads();
#pragma unroll
      for (int t = 0; t < 9; ++t) s_red[tid][t] = dw[t][j];
      __syncthreads();
      if (threadIdx.y == 0 && live) {
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          float a = 0.f;
          for (int y = 0; y < py; ++y) a += s_red[y * cx + threadIdx.x][t];
          atomicAdd(reinterpret_cast<double*>(p.dWt) + (size_t)t * p.C + c + j, (double)a);  // fp64 scratch (cvb_dw_bwd)
        }
      }
    }
    if (p.col_sum && XMODE != CVB_A_RAW) {
#pragma unroll 1
      for (int j = 0; j < 8; ++j) {
        __syncthreads();
        s_red[tid][0] = cs[j];
        s_red[tid][1] = cq[j];
        __syncthreads();
        if (threadIdx.y == 0 && live) {
          float a = 0.f, b = 0.f;
          for (int y = 0; y < py; ++y) { a += s_red[y * cx + threadIdx.x][0]; b += s_red[y * cx + threadIdx.x][1]; }
          atomicAdd(p.col_sum + c + j, (double)a);
          atomicAdd(p.col_sq + c + j, (double)b);
        }
      }
    }
  }
}

void dwd_geometry(int C, int64_t npix, dim3& grid, dim3& block, int& CC) {
  CC = C / 8;
  int cx = 1;
  while (cx < CC && cx < 32) cx <<= 1;  // threadIdx.x spans up to 32 channel chunks (512 B of a pixel row per warp)
  const int py = DNT / cx;
  block = dim3(cx, py, 1);
  int64_t blocks = (npix + py - 1) / py;
  const int64_t cap = 4LL * cvb_num_sms();
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  grid = dim3((unsigned)blocks, 1, 1);
}

}  // namespace

int cvb_dw_fwd_dilated(const cvb_dw_fwd_args& a, cudaStream_t st) {
  CVB_CHECK(a.stride == 1, "cvb_dw_fwd: dilation > 1 needs stride 1 (the reference dilates instead of striding, mobilevit_v2.py:183-186)");
  dim3 grid, block;
  int CC;
  dwd_geometry(a.C, (int64_t)a.B * a.H * a.W, grid, block, CC);
  if (a.x_mode == CVB_A_RAW) CVB_CUDA(cvb_launch(dwd_fwd_kernel<CVB_A_RAW>, grid, block, 0, st, a, a.dilation, CC));
  else if (a.x_mode == CVB_A_AFF) CVB_CUDA(cvb_launch(dwd_fwd_kernel<CVB_A_AFF>, grid, block, 0, st, a, a.dilation, CC));
  else CVB_CUDA(cvb_launch(dwd_fwd_kernel<CVB_A_AFF_SILU>, grid, block, 0, st, a, a.dilation, CC));
  CVB_LAUNCH_CHECK();
  return 0;
}

int cvb_dw_bwd_dilated(const cvb_dw_bwd_args& a, cudaStream_t st) {
  CVB_CHECK(a.stride == 1, "cvb_dw_bwd: dilation > 1 needs stride 1");
  dim3 grid, block;
  int CC;
  dwd_geometry(a.C, (int64_t)a.B * a.H * a.W, grid, block, CC);
  const bool bnb = a.g_mode == CVB_A_BNB;
#define CVB_DWD_BWD(GM)                                                                                                      \
  {                                                                                                                         \
    if (a.x_mode == CVB_A_RAW) CVB_CUDA(cvb_launch(dwd_bwd_kernel<GM, CVB_A_RAW>, grid, block, 0, st, a, a.dilation, CC));    \
    else if (a.x_mode == CVB_A_AFF) CVB_CUDA(cvb_launch(dwd_bwd_kernel<GM, CVB_A_AFF>, grid, block, 0, st, a, a.dilation, CC)); \
    else CVB_CUDA(cvb_launch(dwd_bwd_kernel<GM, CVB_A_AFF_SILU>, grid, block, 0, st, a, a.dilation, CC));                    \
  }
  if (bnb) CVB_DWD_BWD(CVB_A_BNB) else CVB_DWD_BWD(CVB_A_RAW)
#undef CVB_DWD_BWD
  CVB_LAUNCH_CHECK();
  return 0;
}
