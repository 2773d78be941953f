// Validation of the classification recipes (engine/training_engine.py:val_epoch, metrics/topk_accuracy.py,
// loss_fn/classification/cross_entropy.py in eval mode), sm_90a.
//   cvb_cls_metrics : one pass over the classifier's bf16 logits.  Per row: the cross entropy WITHOUT label smoothing (the reference switches
//                     smoothing off in eval mode) and the rank of the target, the number of classes whose logit is STRICTLY greater than the
//                     target's, compared on the bf16 values the classifier wrote (the rule of zs_logits_topk_kernel).  top-k hit iff rank < k,
//                     so a class count below 5 makes every counted row a top-5 hit.  Rows whose target is ignore_index are skipped.
//                     Adds into device accumulators: fp64 sum of the per-row losses and int64 counts {top-1 hits, top-5 hits, rows}.
//                     Deterministic: the counts are integer atomics; the fp32 per-row losses go to caller scratch and the LAST CTA folds
//                     them into fp64 in an order fixed by the row index alone (16-row chunks, chunk c to thread c % 256, threads in order),
//                     so neither the grid nor ignored pad rows (exact zeros) change a bit of the sum.
//   cvb_ema_update  : ema = ema * (1 - m) + m * src over a flat fp32 buffer, in the reference's operation order (averaging_utils.py:55: two
//                     rounded products, one rounded sum; 1 - m is formed in double and rounded to fp32, as torch does with the Python scalar).
#include "common.cuh"

namespace {

constexpr int MT_WARPS = 8;       // rows in flight per CTA: one warp per row
constexpr int MT_MAX_CTAS = 256;
constexpr int FOLD_THREADS = MT_WARPS * 32;
constexpr int FOLD_CHUNK = 16;    // rows per chunk of the final fold

__global__ void __launch_bounds__(MT_WARPS * 32) cls_metrics_kernel(const bf16* __restrict__ logits, int ld, int B, int C,
                                                                    const int64_t* __restrict__ target, int ignore_index, double* loss_sum,
                                                                    unsigned long long* counts, float* row_loss, unsigned int* ticket) {
  __shared__ unsigned int s_cnt[3];
  __shared__ double s_fold[FOLD_THREADS];
  __shared__ unsigned int s_last;
  pdl_wait();
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0u;
  __syncthreads();
  unsigned int top1 = 0u, top5 = 0u, rows = 0u;  // lane 0's tallies
  for (int r = blockIdx.x * MT_WARPS + warp; r < B; r += gridDim.x * MT_WARPS) {
    const int64_t t = target[r];
    float loss = 0.f;
    if (t != (int64_t)ignore_index) {
      const bf16* row = logits + (int64_t)r * ld;
      if (t < 0 || t >= C) {
        loss = __int_as_float(0x7fc00000);  // a label outside [0, C): NaN loss, so it cannot pass unnoticed; the row is a miss
      } else {
        const float xt = __bfloat162float(row[t]);
        float mx = -INFINITY;
        unsigned int above = 0u;
        for (int c = lane; c < C; c += 32) {
          const float v = __bfloat162float(row[c]);
          mx = fmaxf(mx, v);
          above += (v > xt) ? 1u : 0u;
        }
        mx = warp_max(mx);
        above = __reduce_add_sync(0xffffffffu, above);
        float se = 0.f;
        for (int c = lane; c < C; c += 32) se += __expf(__bfloat162float(row[c]) - mx);
        se = warp_sum(se);
        loss = (mx + __logf(se)) - xt;
        top1 += above < 1u ? 1u : 0u;
        top5 += above < 5u ? 1u : 0u;
      }
      rows += 1u;
    }
    if (lane == 0) row_loss[r] = loss;
  }
  if (lane == 0) {
    if (top1) atomicAdd(&s_cnt[0], top1);
    if (top5) atomicAdd(&s_cnt[1], top5);
    if (rows) atomicAdd(&s_cnt[2], rows);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 0; i < 3; ++i)
      if (s_cnt[i]) atomicAdd(counts + i, (unsigned long long)s_cnt[i]);
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  // the last CTA: every row loss is visible (each CTA fenced before taking its ticket); fold them in the row-index order
  __threadfence();
  double acc = 0.0;
  for (int64_t c0 = (int64_t)threadIdx.x * FOLD_CHUNK; c0 < B; c0 += (int64_t)FOLD_THREADS * FOLD_CHUNK)
    for (int j = 0; j < FOLD_CHUNK && c0 + j < B; ++j) acc += (double)__ldcg(row_loss + c0 + j);
  s_fold[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < FOLD_THREADS; ++i) tot += s_fold[i];
    loss_sum[0] += tot;
    *ticket = 0u;  // ready for the next call (and the next replay of a captured graph)
    __threadfence();
  }
}

constexpr int EMA_THREADS = 256;

__global__ void __launch_bounds__(EMA_THREADS) ema_update_kernel(float* __restrict__ ema, const float* __restrict__ src, int64_t n, float keep,
                                                                 float m) {
  pdl_wait();
  pdl_trigger();
  for (int64_t i = (int64_t)blockIdx.x * EMA_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * EMA_THREADS)
    ema[i] = __fadd_rn(__fmul_rn(ema[i], keep), __fmul_rn(m, src[i]));
}

}  // namespace

extern "C" int cvb_cls_metrics(const void* logits, int ld, int B, int C, const int64_t* target, int ignore_index, double* loss_sum,
                               int64_t* counts, float* row_loss, int* ticket, cvb_stream_t stream) {
  CVB_CHECK(logits && target && loss_sum && counts && row_loss && ticket && B > 0 && C > 0 && ld >= C,
            "cvb_cls_metrics: bad arguments (B > 0, C > 0, ld >= C, every pointer given)");
  const int grid = (int)std::min<int64_t>(((int64_t)B + MT_WARPS - 1) / MT_WARPS, MT_MAX_CTAS);
  CVB_CUDA(cvb_launch(cls_metrics_kernel, grid, MT_WARPS * 32, 0, static_cast<cudaStream_t>(stream), static_cast<const bf16*>(logits), ld, B, C,
                      target, ignore_index, loss_sum, reinterpret_cast<unsigned long long*>(counts), row_loss,
                      reinterpret_cast<unsigned int*>(ticket)));
  return 0;
}

extern "C" int cvb_ema_update(float* ema, const float* src, int64_t n, double momentum, cvb_stream_t stream) {
  CVB_CHECK(ema && src && n > 0 && momentum >= 0.0 && momentum <= 1.0, "cvb_ema_update: bad arguments (n > 0, 0 <= momentum <= 1)");
  const int64_t blocks = std::min<int64_t>((n + EMA_THREADS - 1) / EMA_THREADS, (int64_t)cvb_num_sms() * 8);
  CVB_CUDA(cvb_launch(ema_update_kernel, (int)blocks, EMA_THREADS, 0, static_cast<cudaStream_t>(stream), ema, src, n, (float)(1.0 - momentum),
                      (float)momentum));
  return 0;
}
