// Shared by the inference kernels (forward.cu: one CTA per 2*TM detections; forward_small.cu: an 8-CTA cluster per
// 16 detections; forward_wide.cu: the whole grid on one tile of <= 32 detections): kernel parameters, input staging,
// per-row decode and stores.
#pragma once
#include "common.cuh"

namespace mlb {

struct FwdParams {
    const float* blob;
    mlb_op ops[MLB_MAX_OPS];
    int n_ops, in_size, out_size, L, decode_kind;
    int input_kind, flags, n_rows, n_right, n_tiles, kpad0;
    int row_base;  // forward_wide.cu: first row of the single tile this launch processes
    float kinv[9];
    float z_met;
    const float* x;
    const float* xr;
    float* out_raw;
    float* out_dec;
    float* out_xyzc;
    float* out_x;
    const uint8_t* drop_mask;
    unsigned long long drop_seed;
    float p_drop;
    float* res_scratch;
    int* err_flag;
    float* gather[MLB_MAX_PEERS];
    int n_gather;
    long long gather_row0;
    // device-side completion of the fused all-gather (mlb_forward_args.gather_epoch != 0)
    unsigned* gather_flags[MLB_MAX_PEERS];  // rank r's flag array (peer-mapped)
    unsigned gather_epoch;                  // 0: no protocol in this launch
    int gather_rank;
    unsigned* gather_done;                  // this device's monotonic "CTA finished its peer stores" counter
    unsigned gather_done_target;            // its value once every storing CTA of this launch has arrived
};

enum { ERR_GATHER_TIMEOUT = 4 };

// Many images in one launch (mlb_forward_images): the image description, passed as a trailing kernel parameter so that
// no FwdParams field moves.  Only the <IMAGES = true> instantiations read it; the others compile as before.
struct ImgParams {
    const int* row_off;    // [n_img + 1] network rows of image i: [row_off[i], row_off[i + 1])
    const int* left_off;   // stereo: [n_img + 1] offsets into x (left poses)
    const int* right_off;  // stereo: [n_img + 1] offsets into x_right
    const float* kinv;     // [n_img][9] K^-1 row-major
    int n_img, n_left, n_right;  // n_left / n_right: totals over all images (clamp bounds)
};

// Image of network row `grow`: the last i with row_off[i] <= grow, clamped to [0, n_img) whatever the offsets hold.
__device__ __forceinline__ int image_of_row(const ImgParams& ib, int grow) {
    int lo = 0, hi = ib.n_img - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(ib.row_off + mid) <= grow) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Where row `grow` reads its inputs: its image's K^-1 and its left (and right) pose, clamped inside x / x_right.
// Stereo row (l, r) of image i is row_off[i] + l * nr_i + r (the image-local form of the all-vs-all rows l * R + r).
struct RowSrc {
    const float* kinv;
    int li, ri;
};
__device__ __forceinline__ RowSrc row_source(const ImgParams& ib, int grow, bool stereo) {
    const int i = image_of_row(ib, grow);
    RowSrc s;
    s.kinv = ib.kinv + (size_t)i * 9;
    s.li = grow, s.ri = 0;
    if (stereo) {
        const int loc = grow - __ldg(ib.row_off + i);
        const int nr = max(1, __ldg(ib.right_off + i + 1) - __ldg(ib.right_off + i));
        s.li = min(max(__ldg(ib.left_off + i) + loc / nr, 0), ib.n_left - 1);
        s.ri = min(max(__ldg(ib.right_off + i) + loc % nr, 0), ib.n_right - 1);
    }
    return s;
}

// Pre-process of ONE row of a multi-image launch by one thread (process.py:25-67 with the row's own K^-1): the same
// expressions in the same order as the single-K staging code, so a row's network input is bit-identical to that of the
// row run alone with its image's K.  put(k, v) stores input feature k; cen receives (u_c, v_c, x_c * z_met, y_c * z_met).
// A row beyond the batch (live == false) stores zeros.
template <typename Put>
__device__ __forceinline__ void preprocess_row_images(const FwdParams& p, const ImgParams& ib, int grow, bool live, float* cen,
                                                      Put put) {
    const bool stereo = p.input_kind == MLB_IN_KPS_STEREO;
    if (!live) {
        cen[0] = cen[1] = cen[2] = cen[3] = 0.f;
#pragma unroll
        for (int k = 0; k < 34; ++k) put(k, 0.f);
        if (stereo) {
#pragma unroll
            for (int k = 34; k < 68; ++k) put(k, 0.f);
        }
        return;
    }
    const RowSrc s = row_source(ib, grow, stereo);
    const float zm = p.z_met;
    const float k0 = __ldg(s.kinv + 0), k1 = __ldg(s.kinv + 1), k2 = __ldg(s.kinv + 2);
    const float k3 = __ldg(s.kinv + 3), k4 = __ldg(s.kinv + 4), k5 = __ldg(s.kinv + 5);
    const float* kp = p.x + (size_t)s.li * 51;
    const float* kr = p.xr + (size_t)s.ri * 51;
    float umin = __ldg(kp), umax = umin, vmin = __ldg(kp + 17), vmax = vmin;
    for (int j = 1; j < 17; ++j) {
        const float u = __ldg(kp + j), v = __ldg(kp + 17 + j);
        umin = fminf(umin, u), umax = fmaxf(umax, u);
        vmin = fminf(vmin, v), vmax = fmaxf(vmax, v);
    }
    const float uc = __fadd_rn(__fdiv_rn(__fsub_rn(umax, umin), 2.f), umin);  // camera.py:82-86
    const float vc = __fadd_rn(__fdiv_rn(__fsub_rn(vmax, vmin), 2.f), vmin);
    const float cx = (uc * k0 + vc * k1 + k2) * zm, cy = (uc * k3 + vc * k4 + k5) * zm;
    cen[0] = uc, cen[1] = vc, cen[2] = cx, cen[3] = cy;
    const bool zc = (p.flags & MLB_FWD_ZERO_CENTER) != 0;
#pragma unroll
    for (int j = 0; j < 17; ++j) {
        const float u = __ldg(kp + j), v = __ldg(kp + 17 + j);
        float xl = (u * k0 + v * k1 + k2) * zm;  // camera.py:26-27, rows 0/1 of [u v 1] K^-T
        float yl = (u * k3 + v * k4 + k5) * zm;
        if (stereo) {
            const float ur = __ldg(kr + j), vr = __ldg(kr + 17 + j);
            put(34 + 2 * j, xl - (ur * k0 + vr * k1 + k2) * zm);  // process.py:41 cat(l, l - r)
            put(35 + 2 * j, yl - (ur * k3 + vr * k4 + k5) * zm);
        } else if (zc) {
            xl -= cx;  // process.py:61-62
            yl -= cy;
        }
        put(2 * j, xl);
        put(2 * j + 1, yl);
    }
}

// Called by ONE thread of every CTA that stored gather rows, after a CTA barrier that follows those stores.  No per-thread
// fence is needed (one fence.sc.sys per storing thread cost 20 us per launch): the barrier orders the CTA's stores before
// this thread, its gpu-scope fence + arrival (release pattern) and the last arriver's system-scope fence + st.release.sys
// are cumulative over everything observed before them.  The last CTA to arrive publishes this rank's epoch
// into every rank's flag array (release at system scope: cumulativity orders all CTAs' peer stores before the flag) and
// then waits until every rank's epoch has reached this rank's own array -- the kernel retires only when the whole
// gathered buffer is complete here.  Bounded by %globaltimer (20 s): a dead peer raises the error flag instead of hanging.
__device__ __forceinline__ void gather_finish(const FwdParams& p) {
    if (p.n_gather == 0 || p.gather_epoch == 0) return;
    __threadfence();   // gpu scope is enough for the CTA -> last-arriver edge; the last arriver fences at system scope
    const unsigned prev = atomicAdd(p.gather_done, 1u);
    if (prev + 1u != p.gather_done_target) return;
    __threadfence_system();
    for (int r = 0; r < p.n_gather; ++r) {
        unsigned* f = p.gather_flags[r] + (size_t)p.gather_rank * MLB_GATHER_FLAG_STRIDE;
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(f), "r"(p.gather_epoch) : "memory");
    }
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    const unsigned* mine = p.gather_flags[p.gather_rank];
    for (int r = 0; r < p.n_gather; ++r) {
        unsigned spins = 0;
        for (;;) {
            unsigned v;
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine + (size_t)r * MLB_GATHER_FLAG_STRIDE) : "memory");
            if ((int)(v - p.gather_epoch) >= 0) break;
            if ((++spins & 1023u) == 0) {
                unsigned long long t;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
                if (t - t0 > 20000000000ull) {
                    if (p.err_flag) *reinterpret_cast<volatile int*>(p.err_flag) = ERR_GATHER_TIMEOUT;
                    __threadfence_system();
                    return;
                }
            }
        }
    }
    __threadfence_system();
}

// Laplace / spherical / orientation decode of one raw output row (process.py:231-278, 330-360; net.py:95-100).
// Explicit __f*_rn intrinsics pin the reference's operation order (no FMA contraction).
__device__ __forceinline__ void decode_row(int kind, int out_size, const float* o, float& x, float& y, float& z, float& d,
                                           float& bi, float& yaw_p, float& yaw_o, float& aux) {
    x = y = z = d = bi = yaw_p = yaw_o = aux = 0.f;
    if (kind == MLB_DECODE_LOCO) {
        const float th = o[0], ps = o[1];
        d = o[2];
        bi = __fmul_rn(expf(o[3]), d);                    // process.py:132
        x = __fmul_rn(__fmul_rn(d, sinf(ps)), cosf(th));  // camera.py:232
        y = __fmul_rn(d, cosf(ps));                       // camera.py:236
        z = sqrtf(__fsub_rn(__fsub_rn(__fmul_rn(d, d), __fmul_rn(x, x)), __fmul_rn(y, y)));  // process.py:265
        yaw_p = atan2f(o[7], o[8]);                       // process.py:272
        if (out_size == 10) aux = 1.0f / (1.0f + expf(-o[9]));  // process.py:277
    } else if (kind == MLB_DECODE_MONO) {
        x = o[0], y = o[1], z = o[2];
        d = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));  // process.py:350
        bi = __fmul_rn(expf(o[3]), o[2]);
        yaw_p = atan2f(o[7], o[8]);
    } else if (kind == MLB_DECODE_DB) {
        d = o[0];
        bi = __fmul_rn(expf(o[1]), o[0]);  // net.py:98
    }
    if (kind == MLB_DECODE_LOCO || kind == MLB_DECODE_MONO) {
        yaw_o = __fadd_rn(yaw_p, atan2f(x, z));  // camera.py:203-204
        if (yaw_o > 3.14159265358979323846f) yaw_o = __fsub_rn(yaw_o, 6.28318530717958647692f);
        if (yaw_o < -3.14159265358979323846f) yaw_o = __fadd_rn(yaw_o, 6.28318530717958647692f);
    }
}


// Pre-process of one row tile into the k-major input tile xin[k][ld] (process.py:25-67 preprocess_monoloco /
// preprocess_monstereo, camera.py:26-27 pixel_to_camera, camera.py:82-86 bbox centre), rows [row0, row0 + rows_here) ->
// slots 0.., remaining slots and the K padding rows zero.  cen[slot] = (u_c, v_c, x_c * z_met, y_c * z_met).
// `sync` is the caller's barrier over the `nthreads` participating threads.  IMAGES: one thread per row, with the row's
// own K^-1 and poses (preprocess_row_images).
template <bool IMAGES, typename Sync>
__device__ __forceinline__ void stage_input_tile(const FwdParams& p, const ImgParams& ib, int row0, int rows_here, int slots,
                                                 int ld, float* xin, float* cen, int tid, int nthreads, Sync sync) {
    const float zm = p.z_met;
    const float k0 = p.kinv[0], k1 = p.kinv[1], k2 = p.kinv[2], k3 = p.kinv[3], k4 = p.kinv[4], k5 = p.kinv[5];
    if (p.input_kind == MLB_IN_X) {
        for (int idx = tid; idx < slots * p.kpad0; idx += nthreads) {
            const int r = idx / p.kpad0, k = idx % p.kpad0;
            float v = 0.f;
            if (r < rows_here && k < p.in_size) v = __ldg(p.x + (size_t)(row0 + r) * p.in_size + k);
            xin[k * ld + r] = v;
        }
        return;
    }
    if constexpr (IMAGES) {
        for (int r = tid; r < slots; r += nthreads)
            preprocess_row_images(p, ib, row0 + r, r < rows_here, cen + r * 4, [&](int k, float v) { xin[k * ld + r] = v; });
        for (int idx = tid; idx < slots * (p.kpad0 - p.in_size); idx += nthreads)  // zero the K padding rows
            xin[(p.in_size + idx / slots) * ld + idx % slots] = 0.f;
        return;
    }
    const bool stereo = p.input_kind == MLB_IN_KPS_STEREO;
    if (tid < slots) {
        const int r = tid;
        float uc = 0.f, vc = 0.f;
        if (r < rows_here) {
            const float* kp = p.x + (size_t)(stereo ? (row0 + r) / p.n_right : (row0 + r)) * 51;
            float umin = __ldg(kp), umax = umin, vmin = __ldg(kp + 17), vmax = vmin;
            for (int j = 1; j < 17; ++j) {
                const float u = __ldg(kp + j), v = __ldg(kp + 17 + j);
                umin = fminf(umin, u), umax = fmaxf(umax, u);
                vmin = fminf(vmin, v), vmax = fmaxf(vmax, v);
            }
            uc = __fadd_rn(__fdiv_rn(__fsub_rn(umax, umin), 2.f), umin);
            vc = __fadd_rn(__fdiv_rn(__fsub_rn(vmax, vmin), 2.f), vmin);
        }
        cen[r * 4 + 0] = uc;
        cen[r * 4 + 1] = vc;
        cen[r * 4 + 2] = (uc * k0 + vc * k1 + k2) * zm;
        cen[r * 4 + 3] = (uc * k3 + vc * k4 + k5) * zm;
    }
    if (p.flags & MLB_FWD_ZERO_CENTER) sync();
    for (int idx = tid; idx < slots * 17; idx += nthreads) {
        const int r = idx / 17, j = idx % 17;
        float xl = 0.f, yl = 0.f, xd = 0.f, yd = 0.f;
        if (r < rows_here) {
            const int grow = row0 + r;
            const float* kp = p.x + (size_t)(stereo ? grow / p.n_right : grow) * 51;
            const float u = __ldg(kp + j), v = __ldg(kp + 17 + j);
            xl = (u * k0 + v * k1 + k2) * zm;  // rows 0/1 of [u v 1] K^-T
            yl = (u * k3 + v * k4 + k5) * zm;
            if (stereo) {
                const float* kr = p.xr + (size_t)(grow % p.n_right) * 51;
                const float ur = __ldg(kr + j), vr = __ldg(kr + 17 + j);
                xd = xl - (ur * k0 + vr * k1 + k2) * zm;  // process.py:41 cat(l, l - r)
                yd = yl - (ur * k3 + vr * k4 + k5) * zm;
            } else if (p.flags & MLB_FWD_ZERO_CENTER) {
                xl -= cen[r * 4 + 2];  // process.py:61-62
                yl -= cen[r * 4 + 3];
            }
        }
        xin[(2 * j) * ld + r] = xl;
        xin[(2 * j + 1) * ld + r] = yl;
        if (stereo) {
            xin[(34 + 2 * j) * ld + r] = xd;
            xin[(35 + 2 * j) * ld + r] = yd;
        }
    }
    for (int idx = tid; idx < slots * (p.kpad0 - p.in_size); idx += nthreads)  // zero the K padding rows
        xin[(p.in_size + idx / slots) * ld + idx % slots] = 0.f;
}

// One decoded row -> the caller's outputs (raw, decoded, xyz of the bbox-centre ray, fused all-gather peers).
// gather_stage != nullptr: instead of storing the gather row to the peers itself, the row ([MLB_GATHER_LD] floats) is left
// there (shared memory) and the caller ships the whole tile with coalesced stores.
// IMAGES: the bbox-centre ray uses the K^-1 of the row's image (looked up here, once per row) instead of p.kinv.
template <bool IMAGES = false>
__device__ __forceinline__ void store_row(const FwdParams& p, size_t grow, const float* o, const float* cen_row,
                                          float* gather_stage = nullptr, const ImgParams* ib = nullptr) {
    for (int k = 0; k < p.out_size; ++k) p.out_raw[grow * p.out_size + k] = o[k];
    float x, y, z, d, bi, yaw_p, yaw_o, aux;
    decode_row(p.decode_kind, p.out_size, o, x, y, z, d, bi, yaw_p, yaw_o, aux);
    if (p.out_dec != nullptr) {
        float4* dst = reinterpret_cast<float4*>(p.out_dec + grow * 8);
        dst[0] = make_float4(x, y, z, d);
        dst[1] = make_float4(bi, yaw_p, yaw_o, aux);
    }
    if (gather_stage != nullptr) {
        for (int k = 0; k < MLB_GATHER_DEC; ++k) gather_stage[k] = k < p.out_size ? o[k] : 0.f;
        reinterpret_cast<float4*>(gather_stage + MLB_GATHER_DEC)[0] = make_float4(x, y, z, d);
        reinterpret_cast<float4*>(gather_stage + MLB_GATHER_DEC)[1] = make_float4(bi, yaw_p, yaw_o, aux);
    }
    for (int pg = 0; gather_stage == nullptr && pg < p.n_gather; ++pg) {  // the same row straight into every rank's gather buffer over NVLink
        float* dst = p.gather[pg] + (size_t)(p.gather_row0 + (long long)grow) * MLB_GATHER_LD;
        for (int k = 0; k < p.out_size; ++k) dst[k] = o[k];
        reinterpret_cast<float4*>(dst + MLB_GATHER_DEC)[0] = make_float4(x, y, z, d);
        reinterpret_cast<float4*>(dst + MLB_GATHER_DEC)[1] = make_float4(bi, yaw_p, yaw_o, aux);
    }
    if (p.out_xyzc != nullptr && p.input_kind != MLB_IN_X) {
        // net.py:195,213: xy_centers = pixel_to_camera(uv_centers, kk, 1); xyz_from_distance(d, centre)
        const float uc = cen_row[0], vc = cen_row[1];
        float cx, cy, cz;
        if constexpr (IMAGES) {
            const float* kv = ib->kinv + (size_t)image_of_row(*ib, (int)grow) * 9;
            cx = uc * __ldg(kv + 0) + vc * __ldg(kv + 1) + __ldg(kv + 2);
            cy = uc * __ldg(kv + 3) + vc * __ldg(kv + 4) + __ldg(kv + 5);
            cz = uc * __ldg(kv + 6) + vc * __ldg(kv + 7) + __ldg(kv + 8);
        } else {
            cx = uc * p.kinv[0] + vc * p.kinv[1] + p.kinv[2];
            cy = uc * p.kinv[3] + vc * p.kinv[4] + p.kinv[5];
            cz = uc * p.kinv[6] + vc * p.kinv[7] + p.kinv[8];
        }
        const float den = sqrtf(__fadd_rn(__fadd_rn(1.f, __fmul_rn(cx, cx)), __fmul_rn(cy, cy)));
        const float px = __fdiv_rn(__fmul_rn(cx, d), den), py = __fdiv_rn(__fmul_rn(cy, d), den),
                    pz = __fdiv_rn(__fmul_rn(cz, d), den);
        const float nrm = sqrtf(px * px + py * py + pz * pz);
        *reinterpret_cast<float4*>(p.out_xyzc + grow * 4) = make_float4(px, py, pz, nrm);
    }
}

}  // namespace mlb
