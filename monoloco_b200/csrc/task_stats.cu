// Loss statistics of the train / validate / evaluate loop (trainer.py:165-167, 193-197, 250-284) in one launch:
// the MultiTaskLoss train-form total, the CompositeLoss val-form losses and compute_stats' extras for every CSR row
// segment, added into an fp64 accumulator on the device so that an epoch needs no host round trip per batch.
//
// One CTA per segment. Thread t reads rows t, t + 256, ... of its segment and sums them in fp64 in that order; the
// CTA then reduces the 256 partials with a fixed tree and thread 0 adds the result into acc. Nothing depends on timing,
// so two launches on the same inputs give the same bits.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>

#include "../../include/monoloco_b200.h"

extern thread_local std::string g_mlb_err;
void mlb_count_launch();

namespace mlb {

constexpr int STATS_THREADS = 256;
// per-thread partial sums, in this order (the totals are formed from them after the reduction)
enum { P_N, P_VAL, P_BI = P_VAL + 8, P_HIT, P_ERR, P_ERR2, P_MISS, P_LAPLACE, P_ORI_L1, P_COUNT };

__device__ __forceinline__ double bce_logits(double x, double y) {
    // torch binary_cross_entropy_with_logits: (1 - y) x + max(-x, 0) + log(exp(-max) + exp(-x - max))
    const double m = fmax(-x, 0.0);
    return (1.0 - y) * x + m + log(exp(-m) + exp(-x - m));
}

__global__ void __launch_bounds__(STATS_THREADS) task_stats_kernel(const __grid_constant__ mlb_task_stats_args a) {
    const int seg = blockIdx.x;
    const int r0 = a.seg_off[seg], r1 = a.seg_off[seg + 1];
    const int mask = a.task_mask;
    double p[P_COUNT];
#pragma unroll
    for (int k = 0; k < P_COUNT; ++k) p[k] = 0.0;

    for (int r = r0 + (int)threadIdx.x; r < r1; r += STATS_THREADS) {
        const float* o = a.out + (size_t)r * a.out_cols;
        const float* y = a.labels + (size_t)r * a.label_ld;
        const float d = o[2], logb = o[3], d_gt = y[3];
        const float err = fabsf(d - d_gt);
        const float bi = expf(logb) * d;                    // unnormalize_bi, fp32 as in the reference
        p[P_N] += 1.0;
        p[P_BI] += (double)bi;
        p[P_HIT] += err <= bi ? 1.0 : 0.0;
        p[P_ERR] += (double)err;
        p[P_ERR2] += (double)err * (double)err;
        p[P_LAPLACE] += fabs(1.0 - (double)d / (double)d_gt) * exp(-(double)logb) + 0.01 + (double)logb + 2.0;
        p[P_VAL + MLB_TASK_D] += (double)err;               // l1_loss_from_laplace
        p[P_VAL + MLB_TASK_X] += fabs((double)o[0] - (double)y[0]);
        p[P_VAL + MLB_TASK_Y] += fabs((double)o[1] - (double)y[1]);
        p[P_VAL + MLB_TASK_H] += fabs((double)o[4] - (double)y[4]);
        p[P_VAL + MLB_TASK_W] += fabs((double)o[5] - (double)y[5]);
        p[P_VAL + MLB_TASK_L] += fabs((double)o[6] - (double)y[6]);
        p[P_VAL + MLB_TASK_ORI] += fabs(atan2((double)o[7], (double)o[8]) - atan2((double)y[7], (double)y[8]));
        p[P_ORI_L1] += fabs((double)o[7] - (double)y[7]) + fabs((double)o[8] - (double)y[8]);
        if (mask & (1 << MLB_TASK_AUX)) {
            const float x = o[9], t = y[10];
            p[P_VAL + MLB_TASK_AUX] += bce_logits((double)x, (double)t);
            const float sig = 1.0f / (1.0f + expf(-x));
            p[P_MISS] += fabs((sig >= 0.5f ? 1.0 : 0.0) - (double)t);
        }
    }

    // fixed-order tree over the CTA: warp shuffles (xor pattern), then the 8 warp sums by warp 0
    __shared__ double red[STATS_THREADS / 32][P_COUNT];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < P_COUNT; ++k) {
        double v = p[k];
        for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
        if (lane == 0) red[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    double s[P_COUNT];
    for (int k = 0; k < P_COUNT; ++k) {
        double v = 0.0;
        for (int w = 0; w < STATS_THREADS / 32; ++w) v += red[w][k];
        s[k] = v;
    }
    const double n = s[P_N];
    double* acc = a.acc + (size_t)seg * MLB_STATS_NACC;
    if (n == 0.0) return;
    // train-form total: rows * (sum_t w_t mean_t + sum log_sigma); the ori L1 mean runs over 2 * rows elements
    double total = 0.0, sum_ls = 0.0;
    int i = 0;
    for (int t = 0; t < 8; ++t) {
        if (!(mask & (1 << t))) continue;
        double w = (double)a.lambdas[t];
        if (a.log_sigmas) {
            const double ls = (double)a.log_sigmas[i];
            const double e = exp(ls);
            w = w / (2.0 * (e * e));
            sum_ls += ls;
        }
        const double sum_t = t == MLB_TASK_D ? s[P_LAPLACE] : t == MLB_TASK_ORI ? 0.5 * s[P_ORI_L1] : s[P_VAL + t];
        total += w * sum_t;
        ++i;
    }
    total += n * sum_ls;
    acc[MLB_STAT_N] += n;
    acc[MLB_STAT_TOTAL] += total;
    for (int t = 0; t < 8; ++t)
        if (mask & (1 << t)) acc[MLB_STAT_VAL + t] += s[P_VAL + t];
    acc[MLB_STAT_BI] += s[P_BI];
    acc[MLB_STAT_BI_HIT] += s[P_HIT];
    acc[MLB_STAT_ERR] += s[P_ERR];
    acc[MLB_STAT_ERR2] += s[P_ERR2];
    if (mask & (1 << MLB_TASK_AUX)) acc[MLB_STAT_AUX_MISS] += s[P_MISS];
    acc[MLB_STAT_LAPLACE] += s[P_LAPLACE];
    acc[MLB_STAT_ORI_L1] += s[P_ORI_L1];
}

}  // namespace mlb

static int stats_fail(const std::string& msg) {
    g_mlb_err = "mlb_task_stats: " + msg;
    return -1;
}

extern "C" int mlb_task_stats(const mlb_task_stats_args* args, void* stream) {
    if (!args) return stats_fail("args is NULL");
    const mlb_task_stats_args& a = *args;
    if (a.n_seg < 1 || a.n_seg > MLB_STATS_MAX_SEG)
        return stats_fail("n_seg must be in [1, " + std::to_string(MLB_STATS_MAX_SEG) + "] (got " + std::to_string(a.n_seg) + ")");
    if (a.task_mask <= 0 || (a.task_mask & ~0xff))
        return stats_fail("task_mask " + std::to_string(a.task_mask) + " names no task or an unknown one (bits 0..7 only)");
    if (a.out_cols != 9 && a.out_cols != 10)
        return stats_fail("out_cols must be 9 (mono) or 10 (stereo) (got " + std::to_string(a.out_cols) + ")");
    if (a.label_ld != 10 && a.label_ld != 11)
        return stats_fail("label_ld must be 10 (mono) or 11 (stereo) (got " + std::to_string(a.label_ld) + ")");
    if ((a.task_mask & (1 << MLB_TASK_AUX)) && (a.out_cols != 10 || a.label_ld != 11))
        return stats_fail("the aux task needs out_cols = 10 and label_ld = 11");
    if (a.reserved != 0) return stats_fail("reserved must be 0");
    if (a.seg_off[0] < 0) return stats_fail("seg_off[0] must be >= 0");
    for (int s = 0; s < a.n_seg; ++s)
        if (a.seg_off[s + 1] < a.seg_off[s])
            return stats_fail("seg_off must be non-decreasing (seg_off[" + std::to_string(s + 1) + "] = " +
                              std::to_string(a.seg_off[s + 1]) + " < " + std::to_string(a.seg_off[s]) + ")");
    if (!a.acc) return stats_fail("acc is NULL");
    if (a.seg_off[a.n_seg] > 0 && (!a.out || !a.labels)) return stats_fail("out or labels is NULL");
    mlb::task_stats_kernel<<<a.n_seg, mlb::STATS_THREADS, 0, (cudaStream_t)stream>>>(a);
    mlb_count_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return stats_fail(cudaGetErrorString(e));
    return 0;
}
