// monoloco_b200 -- activity heuristics after post-processing, for many images in one launch:
//
//   * social distancing / F-formation   monoloco/activity.py:17-67 (social_interactions), :120-165 (check_f_formations)
//   * raised hand                       monoloco/activity.py:70-117 (is_raising_hand)
//
// The flags are decisions on geometry, so every expression follows the reference's arithmetic exactly:
//   * Python floats / numpy fp64 -> explicit __d*_rn; the 1-D np.linalg.norm of a 2-vector is sqrt(fma(b, b, a * a)),
//     the row-wise norm (axis=1) is sqrt(a * a + b * b), np.dot of two 2-vectors is fma(a1, b1, a0 * b0);
//   * torch fp32 tensors (dds, stds, the draws and the moved centre) -> explicit __f*_rn;
//   * the Laplace draws are dds[p] - |stds[p]| * T[s * n + p]: T = sign(u) * log1p(-|u|) of torch's seed-1 CPU stream,
//     computed by torch on the host (a device log1pf does not round like torch's), so only the fp32 fmul / fsub remain.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <string>

#include "../../include/monoloco_b200.h"

extern thread_local std::string g_mlb_err;
void mlb_count_launch();

namespace mlb_act {

struct Person {   // one person of the image being processed, in shared memory
    double x, z;  // centre
    double ca, sa;  // cos / sin of the orientation (the o-space candidate, activity.py:138-143)
    float cr, sr;   // fp32 cos / sin of the centre ray atan2(z, x) (the moved centre, activity.py:57-59)
    float dd, b;    // d and |std|, fp32 (torch.tensor(dds), torch.abs(stds))
};

__device__ __forceinline__ double norm_fma(double a, double b) { return __dsqrt_rn(__fma_rn(b, b, __dmul_rn(a, a))); }
__device__ __forceinline__ double norm_rows(double a, double b) {
    return __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));
}

// check_f_formations(idx, jdx, centers, ...) with the (possibly moved) centres of the two people; everybody else unmoved
__device__ bool f_formation(const Person* P, int m, int idx, int jdx, double xi, double zi, double xj, double zj,
                            const mlb_social_args& a) {
    for (int r = 0; r < a.n_radii; ++r) {
        const double rad = a.radii[r];
        const double m0x = __dadd_rn(xi, __dmul_rn(rad, P[idx].ca)), m0z = __dsub_rn(zi, __dmul_rn(rad, P[idx].sa));
        const double m1x = __dadd_rn(xj, __dmul_rn(rad, P[jdx].ca)), m1z = __dsub_rn(zj, __dmul_rn(rad, P[jdx].sa));
        const double ocx = __ddiv_rn(__dadd_rn(m0x, m1x), 2.0), ocz = __ddiv_rn(__dadd_rn(m0z, m1z), 2.0);
        double d_new = norm_fma(__dsub_rn(m0x, m1x), __dsub_rn(m0z, m1z));
        if (a.social_distance) d_new = __ddiv_rn(d_new, 2.0);
        const double d0 = norm_fma(__dsub_rn(xi, ocx), __dsub_rn(zi, ocz));
        const double d1 = norm_fma(__dsub_rn(xj, ocx), __dsub_rn(zj, ocz));
        const double dmin = d1 < d0 ? d1 : d0;  // Python min(d_0, d_1)
        if (!(d_new <= dmin)) continue;
        // np.min(other_distances) > radius: every other person strictly outside (a NaN distance makes the min NaN)
        bool clear = true, any = false;
        for (int k = 0; k < m && clear; ++k) {
            if (k == idx || k == jdx) continue;
            any = true;
            clear = norm_rows(__dsub_rn(P[k].x, ocx), __dsub_rn(P[k].z, ocz)) > rad;
        }
        if (!any) clear = 100.0 > rad;  // nobody else: the literal 100 (activity.py:158-159)
        if (clear) return true;
    }
    return false;
}

// new_centers[el] += (dds[el] - sample) * (cos, sin)(atan2(z, x)), in fp32 on torch tensors (activity.py:55-61)
__device__ __forceinline__ void move(float delta, float cr, float sr, double& x, double& z) {
    const float nx = __fadd_rn(__fmul_rn(delta, cr), (float)x);
    const float nz = __fadd_rn(__fmul_rn(delta, sr), (float)z);
    x = nx, z = nz;
}

__global__ void __launch_bounds__(256) social_kernel(const mlb_social_args a) {
    extern __shared__ __align__(16) unsigned char sm_act[];
    Person* P = reinterpret_cast<Person*>(sm_act);
    int* drop = reinterpret_cast<int*>(P + a.max_people);  // first index of argsort(distances) (dropped, :28-30)
    volatile int* flag = drop + a.max_people;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
    const bool prob = a.n_samples >= 2;
    const int n_eval = prob ? a.n_samples : 1;

    for (int img = blockIdx.x; img < a.n_img; img += gridDim.x) {
        const int p0 = min(max(a.img_off[img], 0), a.n_people);
        const int p1 = min(max(a.img_off[img + 1], p0), a.n_people);
        const int m = min(p1 - p0, a.max_people);
        for (int p = tid; p < m; p += blockDim.x) {
            Person q;
            q.x = a.xz[2 * (size_t)(p0 + p)], q.z = a.xz[2 * (size_t)(p0 + p) + 1];
            const double ang = a.angles[p0 + p];
            q.ca = cos(ang), q.sa = sin(ang);
            const double th = atan2(q.z, q.x);
            q.cr = (float)cos(th), q.sr = (float)sin(th);
            q.dd = prob ? a.dds[p0 + p] : 0.f;
            q.b = prob ? fabsf(a.stds[p0 + p]) : 0.f;
            P[p] = q;
            flag[p] = 0;
        }
        for (int p = p0 + m + tid; p < p1; p += blockDim.x) a.out[p] = 0;  // beyond max_people: not evaluated
        __syncthreads();
        // np.argsort(distances)[0]: distance 0 is the minimum (the person itself), ties in index order
        for (int p = tid; p < m; p += blockDim.x) {
            int k = 0;
            for (; k < m; ++k)
                if (norm_rows(__dsub_rn(P[p].x, P[k].x), __dsub_rn(P[p].z, P[k].z)) == 0.0) break;
            drop[p] = k;
        }
        __syncthreads();
        // one warp per (person, neighbour) pair
        for (int pair = warp; pair < m * m; pair += n_warps) {
            const int idx = pair / m, jdx = pair - idx * m;
            if (__shfl_sync(0xffffffffu, flag[idx], 0) || jdx == drop[idx]) continue;  // warp-uniform read
            const double dist = norm_rows(__dsub_rn(P[idx].x, P[jdx].x), __dsub_rn(P[idx].z, P[jdx].z));
            if (!(dist <= a.threshold_dist)) continue;
            int hits = 0;
            for (int s0 = 0; s0 < n_eval; s0 += 32) {
                const int s = s0 + lane;
                bool hit = false;
                if (s < n_eval) {
                    double xi = P[idx].x, zi = P[idx].z, xj = P[jdx].x, zj = P[jdx].z;
                    if (prob) {
                        const Person& pi = P[idx];
                        const float ti = a.table[(size_t)s * m + idx];
                        const float di = __fsub_rn(pi.dd, __fsub_rn(pi.dd, __fmul_rn(pi.b, ti)));
                        move(di, pi.cr, pi.sr, xi, zi);
                        if (jdx == idx) {  // the same person twice (coincident centres): the second step starts moved
                            const double th = atan2(zi, xi);
                            move(di, (float)cos(th), (float)sin(th), xi, zi);
                            xj = xi, zj = zi;
                        } else {
                            const Person& pj = P[jdx];
                            const float tj = a.table[(size_t)s * m + jdx];
                            move(__fsub_rn(pj.dd, __fsub_rn(pj.dd, __fmul_rn(pj.b, tj))), pj.cr, pj.sr, xj, zj);
                        }
                    }
                    hit = f_formation(P, m, idx, jdx, xi, zi, xj, zj, a);
                }
                hits += __popc(__ballot_sync(0xffffffffu, hit));
                // sum(f_forms) / n_samples >= threshold_prob; hits only grow, so the decision is final once it holds
                const bool yes = prob ? __ddiv_rn((double)hits, (double)a.n_samples) >= a.threshold_prob : hits > 0;
                if (yes) {
                    if (lane == 0) flag[idx] = 1;
                    break;
                }
            }
        }
        __syncthreads();
        for (int p = tid; p < m; p += blockDim.x) a.out[p0 + p] = (uint8_t)flag[p];
        __syncthreads();
    }
}

// is_raising_hand, one side: up, elbow angle >= 30 in the reference's (90 / pi) units, not tucked next to the head
__device__ __forceinline__ bool arm_risen(const double* X, const double* Y, int sho, int elb, int hand, double head_top,
                                          bool left) {
    const double f0 = __dsub_rn(X[hand], X[elb]), f1 = __dsub_rn(Y[hand], Y[elb]);
    const double a0 = __dsub_rn(X[sho], X[elb]), a1 = __dsub_rn(Y[sho], Y[elb]);
    const double nf = norm_fma(f0, f1), na = norm_fma(a0, a1);
    const double c = __fma_rn(__ddiv_rn(f1, nf), __ddiv_rn(a1, na), __dmul_rn(__ddiv_rn(f0, nf), __ddiv_rn(a0, na)));
    const double angle = __dmul_rn(90.0 / 3.141592653589793, acos(c));  // NaN (zero-length limb, |c| > 1): not risen
    const bool up = Y[hand] < Y[sho];
    const bool tucked = (left ? X[hand] <= X[sho] : X[hand] >= X[sho]) && Y[hand] >= head_top;
    return up && angle >= 30.0 && !tucked;
}

__global__ void raising_hand_kernel(const double* __restrict__ kps, int n, int8_t* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* X = kps + (size_t)i * 51;
    const double* Y = X + 17;
    const double head_top = __dsub_rn(Y[0], __dsub_rn(X[3], X[4]));  // nose y - (l_ear x - r_ear x)
    const bool l = arm_risen(X, Y, 5, 7, 9, head_top, true), r = arm_risen(X, Y, 6, 8, 10, head_top, false);
    out[i] = (int8_t)(l && r ? 3 : (l ? 1 : (r ? 2 : 0)));
}

}  // namespace mlb_act

using namespace mlb_act;

static int afail(const std::string& msg) {
    g_mlb_err = msg;
    return -1;
}

extern "C" int mlb_social_distance(const mlb_social_args* a, void* stream) {
    if (!a) return afail("mlb_social_distance: null argument");
    if (a->n_img < 1) return afail("mlb_social_distance: n_img must be >= 1");
    if (a->n_people < 0) return afail("mlb_social_distance: negative n_people");
    if (a->max_people < 0 || a->max_people > MLB_SOCIAL_MAX_PEOPLE)
        return afail("mlb_social_distance: max_people " + std::to_string(a->max_people) + " outside 0.." +
                     std::to_string(MLB_SOCIAL_MAX_PEOPLE) + " (people per image)");
    if (a->n_radii < 1 || a->n_radii > MLB_SOCIAL_MAX_RADII) return afail("mlb_social_distance: n_radii must be 1..8");
    if (!a->img_off || !a->xz || !a->angles || !a->out) return afail("mlb_social_distance: null pointer");
    const bool prob = a->n_samples >= 2;
    if (prob && (!a->dds || !a->stds || !a->table)) return afail("mlb_social_distance: null pointer (dds / stds / table)");
    if (prob && a->table_len < (int64_t)a->n_samples * a->max_people)
        return afail("mlb_social_distance: draw table shorter than n_samples * max_people");
    if (a->n_people == 0) return 0;
    const size_t smem = (size_t)a->max_people * (sizeof(Person) + 2 * sizeof(int));
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(social_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return afail(std::string("mlb_social_distance: ") + cudaGetErrorString(e));
    }
    const int grid = a->n_img < 65535 ? a->n_img : 65535;
    social_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(*a);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return afail(std::string("mlb_social_distance: ") + cudaGetErrorString(e));
    mlb_count_launch();
    return 0;
}

extern "C" int mlb_raising_hand(const double* kps, int n, int8_t* out, void* stream) {
    if (n < 0) return afail("mlb_raising_hand: negative n");
    if (n == 0) return 0;
    if (!kps || !out) return afail("mlb_raising_hand: null pointer");
    raising_hand_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(kps, n, out);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return afail(std::string("mlb_raising_hand: ") + cudaGetErrorString(e));
    mlb_count_launch();
    return 0;
}
