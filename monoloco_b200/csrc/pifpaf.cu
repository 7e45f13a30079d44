// monoloco_b200 -- preprocess_pifpaf (monoloco/network/process.py:155-207) for all annotations of all images in one launch.
//
// One CTA per image (CSR offsets over the annotations).  Every number is a Python float in the reference, so every
// expression is fp64 with explicit __d*_rn in the reference's operation order:
//   * with a score:    conf = score, delta_h = h / (10 * enlarge), delta_w = w / (5 * enlarge), xywh -> corners;
//   * without a score: conf = float(np.mean(confs)) in numpy's pairwise order for 17 values (eight accumulators
//                      r[j] = c[j] + c[8 + j], ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), + c[16], / 17),
//                      delta_h = (y2 - y1) / (7 * enlarge), delta_w = (x2 - x1) / (3.5 * enlarge), and the reference's
//                      `assert delta_h > -5 and delta_w > -5` becomes bit 0 of the error word;
//   * clamping with Python's argument order: max(0, v) is v only when v > 0, min(v, size) is size only when size < v
//     (a NaN coordinate becomes 0 on the low side and stays NaN on the high side, as in the reference).
// Kept annotations (conf >= min_conf) are compacted image-major, each image in its original order.  The images' kept
// offsets come from a single-pass chained scan: CTAs take their image from a ticket counter (so every image a CTA waits
// for belongs to a CTA that is already running), publish their kept count at once and their inclusive prefix as soon as
// they know it, and look back over their predecessors until they meet an inclusive prefix.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>

#include "../../include/monoloco_b200.h"

extern thread_local std::string g_mlb_err;
void mlb_count_launch();

namespace mlb_pif {

constexpr int kThreads = 128;
constexpr unsigned long long kAggregate = 1ull << 62;   // state word: count of this image alone
constexpr unsigned long long kInclusive = 2ull << 62;   // state word: kept rows of this image and all before it
constexpr unsigned long long kValueMask = 0xffffffffull;
constexpr unsigned long long kLookbackTimeoutNs = 2000000000ull;

__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// box x1 y1 x2 y2 and conf of annotation k of image img; returns the reference's assert as `bad`
__device__ void annotation(const mlb_pifpaf_args& a, int img, int k, double box[4], double& conf, bool& bad) {
    const double* kp = a.kps + (size_t)k * 51;
    const double* bb = a.bbox + (size_t)k * 4;
    double x1 = bb[0], y1 = bb[1], x2 = bb[2], y2 = bb[3], dh, dw;
    bad = false;
    if (a.has_score != nullptr && a.has_score[k]) {
        conf = a.score[k];
        dh = __ddiv_rn(y2, 10.0 * a.enlarge);
        dw = __ddiv_rn(x2, 5.0 * a.enlarge);
        x2 = __dadd_rn(x2, x1);
        y2 = __dadd_rn(y2, y1);
    } else {
        double r[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(kp[3 * j + 2], kp[3 * (8 + j) + 2]);
        const double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                                   __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
        conf = __ddiv_rn(__dadd_rn(s, kp[3 * 16 + 2]), 17.0);
        dh = __ddiv_rn(__dsub_rn(y2, y1), 7.0 * a.enlarge);
        dw = __ddiv_rn(__dsub_rn(x2, x1), 3.5 * a.enlarge);
        bad = !(dh > -5.0 && dw > -5.0);
    }
    x1 = __dsub_rn(x1, dw);
    y1 = __dsub_rn(y1, dh);
    x2 = __dadd_rn(x2, dw);
    y2 = __dadd_rn(y2, dh);
    if (a.has_size != nullptr && a.has_size[img]) {
        const double w = a.im_size[2 * (size_t)img], h = a.im_size[2 * (size_t)img + 1];
        x1 = x1 > 0.0 ? x1 : 0.0;
        y1 = y1 > 0.0 ? y1 : 0.0;
        x2 = w < x2 ? w : x2;
        y2 = h < y2 ? h : y2;
    }
    box[0] = x1, box[1] = y1, box[2] = x2, box[3] = y2;
}

__global__ void __launch_bounds__(kThreads) pifpaf_kernel(const mlb_pifpaf_args a) {
    __shared__ int s_img, s_warp[kThreads / 32];
    __shared__ long long s_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned long long* state = reinterpret_cast<unsigned long long*>(a.scratch);   // [n_img]
    unsigned int* ticket = reinterpret_cast<unsigned int*>(state + a.n_img);
    if (tid == 0) s_img = (int)atomicAdd(ticket, 1u);
    __syncthreads();
    const int img = s_img;
    const int k0 = min(max(a.ann_off[img], 0), a.n_ann), k1 = min(max(a.ann_off[img + 1], k0), a.n_ann);

    // pass 1: kept count of this image (and the degenerate-box check, which precedes the filter in the reference)
    int mine = 0;
    bool bad_any = false;
    for (int k = k0 + tid; k < k1; k += kThreads) {
        double box[4], conf;
        bool bad;
        annotation(a, img, k, box, conf, bad);
        mine += conf >= a.min_conf;
        bad_any |= bad;
    }
    if (bad_any) atomicOr(a.error, 1);
    for (int s = 16; s > 0; s >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, s);
    if (lane == 0) s_warp[warp] = mine;
    __syncthreads();
    if (tid == 0) {
        long long count = 0;
        for (int w = 0; w < kThreads / 32; ++w) count += s_warp[w];
        long long base = 0;
        if (img > 0) {
            atomicExch(&state[img], kAggregate | (unsigned long long)count);
            const unsigned long long t0 = global_ns();
            for (int j = img - 1; j >= 0;) {
                const unsigned long long s = *reinterpret_cast<volatile unsigned long long*>(&state[j]);
                if (s == 0) {
                    if (global_ns() - t0 > kLookbackTimeoutNs) {
                        atomicOr(a.error, 2);
                        break;
                    }
                    continue;
                }
                base += (long long)(s & kValueMask);
                if (s & kInclusive) break;
                --j;
            }
        }
        atomicExch(&state[img], kInclusive | (unsigned long long)(base + count));
        a.kept_off[img + 1] = (int32_t)(base + count);
        if (img == 0) a.kept_off[0] = 0;
        s_base = base;
    }
    __syncthreads();

    // pass 2: compact the kept annotations in their original order (one ballot scan per chunk of kThreads)
    long long next = s_base;
    for (int c0 = k0; c0 < k1; c0 += kThreads) {
        const int k = c0 + tid;
        double box[4], conf = 0.0;
        bool bad, keep = false;
        if (k < k1) {
            annotation(a, img, k, box, conf, bad);
            keep = conf >= a.min_conf;
        }
        const unsigned int ballot = __ballot_sync(0xffffffffu, keep);
        __syncthreads();   // s_warp of the previous chunk has been read by everybody
        if (lane == 0) s_warp[warp] = __popc(ballot);
        __syncthreads();
        long long pos = next + __popc(ballot & ((1u << lane) - 1u));
        int total = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
            if (w < warp) pos += s_warp[w];
            total += s_warp[w];
        }
        if (keep) {
            double* ob = a.out_boxes + (size_t)pos * 5;
            ob[0] = box[0], ob[1] = box[1], ob[2] = box[2], ob[3] = box[3], ob[4] = conf;
            const double* kp = a.kps + (size_t)k * 51;
            double* o64 = a.out_kps + (size_t)pos * 51;
            float* o32 = a.out_kps32 + (size_t)pos * 51;
            for (int t = 0; t < 17; ++t)
                for (int c = 0; c < 3; ++c) {   // [3][17] rows x, y, conf (prepare_pif_kps, process.py:208-216)
                    const double v = kp[3 * t + c];
                    o64[c * 17 + t] = v;
                    o32[c * 17 + t] = (float)v;
                }
            a.out_src[pos] = k;
        }
        next += total;
    }
}

}  // namespace mlb_pif

using namespace mlb_pif;

static int pif_fail(const std::string& msg) {
    g_mlb_err = "mlb_preprocess_pifpaf: " + msg;
    return -1;
}

extern "C" int mlb_preprocess_pifpaf(const mlb_pifpaf_args* a, void* stream) {
    if (!a) return pif_fail("null argument");
    if (a->n_img < 1) return pif_fail("n_img must be >= 1");
    if (a->n_ann < 0) return pif_fail("negative n_ann");
    if (a->enlarge != 1 && a->enlarge != 2) return pif_fail("enlarge must be 1 or 2");
    if (!isfinite(a->min_conf)) return pif_fail("min_conf must be finite");
    if (!a->ann_off || !a->kept_off || !a->error || !a->scratch) return pif_fail("null pointer");
    if (a->n_ann > 0 && (!a->kps || !a->bbox || !a->out_boxes || !a->out_kps || !a->out_kps32 || !a->out_src))
        return pif_fail("null pointer");
    if (a->has_score && !a->score) return pif_fail("has_score without score");
    if (a->has_size && !a->im_size) return pif_fail("has_size without im_size");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(a->scratch, 0, ((size_t)a->n_img + 1) * sizeof(uint64_t), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(a->error, 0, sizeof(int32_t), st);
    if (e != cudaSuccess) return pif_fail(cudaGetErrorString(e));
    pifpaf_kernel<<<a->n_img, kThreads, 0, st>>>(*a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return pif_fail(cudaGetErrorString(e));
    mlb_count_launch();
    return 0;
}
