// monoloco_b200 -- throughput kernel on the Hopper tensor cores: the fp32 network as error-compensated TF32 products.
//
// The 1e-5 parity rule excludes plain TF32 / BF16 (SURVEY.md §0.4).  Here every fp32 operand is split into two TF32 terms,
// a = a_hi + a_lo (cvt.rna twice), and each layer product runs as THREE wgmma.mma_async tf32 products: a_hi.w_hi into a main
// register accumulator, a_lo.w_hi + a_hi.w_lo into a second one (the dropped a_lo.w_lo term is 2^-22 relative).  The two
// accumulators are added once per layer, in fp32, before the epilogue (tests force this kernel on every fixture).
//
// Replaces, like forward.cu, in ONE launch per detection batch (reference file:line):
//   monoloco/network/process.py:25-67 (pre-process), architectures.py:48-71 / 88-102 / 135-145 (network),
//   process.py:231-278, 330-360 + utils/camera.py:161-177, 202-237 (decode, xyz_from_distance).
//
//   weights      re-packed once per model: per GEMM op  [L/256 column tiles][K/16 k blocks][hi | lo][256 x 16]  (canonical
//                K-major no-swizzle GMMA layout: core matrix 8 rows x 16 B, SBO 128 B, LBO rows x 16 B) -> a pipeline stage
//                is two 1-D TMA bulk copies (8 KB of X planes + 32 KB of W planes), no tensor maps
//   kernel       one cooperative, persistent grid of CTA groups, L/256 CTAs each (4 at L = 1024; floor(SMs / (L/256)) groups,
//                33 on a 132-SM H100).  A group owns a private workspace slot (input planes, two ping-pong activation plane
//                sets, the fp32 residual, the head partials, its barrier counter) and walks 64-row tiles.  CTA n owns output
//                columns [256n, 256n + 256) of every layer.  Groups are not hardware clusters: clusters must fit one GPC,
//                and only 30 four-CTA clusters fit an H100 at once (120 of 132 SMs; a 4096 batch then takes three rounds
//                of tiles instead of two).
//   per tile     prologue: thread = row: pre-process the raw keypoints (process.py:47-67 / 25-44) straight into hi / lo planes
//                per layer: the producer lane streams the stages through a 4-slot ring, running ahead of the consumers
//                within a tile (a layer's W planes while the previous layer finishes, its X planes once the group barrier
//                publishes them) and bulk-copies the layer's epilogue constants into one of two buffers; consumer
//                warpgroup c issues 2 k-steps x 3 wgmma (M 64, N 128, K 8) per stage on output columns [128c, 128c + 128)
//                and releases the stage once its wgmma group retired.
//                Two 64 x 128 accumulators per warpgroup = 128 registers per thread: a 128-row tile would need twice that.
//                The summed accumulators go through shared memory (the layer's last two ring slots, held until read) to a
//                thread = (row, 64 columns) epilogue:
//                folded BN / ReLU / dropout / residual, written straight into the next layer's hi / lo planes; narrow heads
//                (w_aux, w_fin, MonolocoModel.w2) are accumulated on the CUDA cores from the same registers;
//                a group barrier (tc_group_sync: counter in global memory) separates the layers
//   tail         head partial sums -> the group slot -> CTA 0 (fixed summation order) -> decode_row -> stores (raw, decoded,
//                xyz of the bbox-centre ray, fused all-gather peers), exactly the epilogue of the FFMA kernels (fwd_common.cuh).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <string>

#include "fwd_common.cuh"

namespace mlb {

constexpr int TCM = 64, TCN = 256, TCKB = 16, TCNST = 4;   // row tile, columns per CTA, k block, ring
constexpr int TCWN = 128;          // output columns per consumer warpgroup (wgmma N)
constexpr int TCH = 64;            // output columns per epilogue thread
constexpr uint32_t TC_A_PLANE = TCM * TCKB * 4;   // bytes of one X plane block (64 rows x 16 k)
constexpr uint32_t TC_W_PLANE = TCN * TCKB * 4;   // bytes of one W plane block (256 output columns x 16 k)
constexpr uint32_t TC_STAGE = 2 * TC_A_PLANE + 2 * TC_W_PLANE;   // 40 KB: X hi|lo + W hi|lo
constexpr uint32_t TC_LBO_A = TCM * 16, TC_LBO_W = TCN * 16, TC_SBO = 128;
constexpr int TC_MAX_CT = 8;       // column tiles = CTAs per group (L <= 2048)
constexpr int TC_HW = 16;          // head output columns in total (output_size <= 16)
constexpr int TC_EPI = 256;        // consumer threads: 2 warpgroups (wgmma), then the epilogue, thread = (row, 64 columns)
constexpr int TC_THREADS = TC_EPI + 32;   // + the producer warp (TMA ring, epilogue constants)
constexpr int TC_SLD = TCWN + 8;   // row stride (floats) of a warpgroup's staging tile: conflict-free float2 stores
constexpr size_t TC_RING_BYTES = (size_t)TCNST * TC_STAGE;                      // 160 KB
constexpr size_t TC_SST_BYTES = 2 * TCN * sizeof(float);                        // folded-BN scale | shift of the layer
constexpr size_t TC_HW_BYTES = (size_t)TC_HW * TCN * sizeof(float);             // head weights of the layer
constexpr size_t TC_CONST_BYTES = TC_SST_BYTES + TC_HW_BYTES;                   // one buffer of epilogue constants
constexpr size_t TC_SMEM_BYTES = TC_RING_BYTES + 2 * TC_CONST_BYTES;            // 196 KB: two constant buffers
static_assert((size_t)TCM * TC_SLD * sizeof(float) <= TC_STAGE, "a warpgroup's staging tile fits one ring slot");
static_assert((size_t)4 * TC_MAX_CT * TCM * TC_HW * sizeof(float) <= TC_RING_BYTES, "head partials alias the ring");

struct TcExtra {
    const float* wplanes[MLB_MAX_OPS];  // per GEMM op: [L/256 column tiles][n_kb][hi|lo][256 x 16]
    int n_kb[MLB_MAX_OPS];              // K blocks of 16 (K zero-padded)
    float* ws;                          // workspace, one slot per group
    unsigned long long slot_floats;
    int n_tiles;                        // 64-row tiles of this launch
    // narrow heads: rows of all head ops concatenated (q = 0 .. n_head_rows-1)
    int n_head_rows;
    int head_src[TC_HW];                // op index of the GEMM whose output head row q reads
    int head_col[TC_HW];                // raw output column of head row q
    long long head_w[TC_HW];            // float offset of head row q's K weights in the blob
    long long head_b[TC_HW];            // float offset of its bias
};

__device__ __forceinline__ float tc_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
// shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor): start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46),
// base offset 0 [49,52), layout type INTERLEAVE (no swizzle) [62,64)
__device__ __forceinline__ uint64_t tc_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
    uint64_t d = (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((TC_SBO >> 4) & 0x3FFFu) << 32;
    return d;
}
// D[64 x 128] += A[64 x 8] . B[128 x 8]^T, both operands K-major tf32 in shared memory, issued by the whole warpgroup
__device__ __forceinline__ void tc_wgmma(float* d, uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1;\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc));
}
__device__ __forceinline__ void tc_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tc_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous wgmma window
__device__ __forceinline__ void tc_fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < TCWN / 2; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void tc_consumer_sync() { asm volatile("bar.sync 2, 256;" ::: "memory"); }   // the 2 consumer warpgroups
__device__ __forceinline__ void tc_warpgroup_sync(int wg) {   // one consumer warpgroup (named barriers 3 and 4)
    if (wg == 0) asm volatile("bar.sync 3, 128;" ::: "memory");
    else asm volatile("bar.sync 4, 128;" ::: "memory");
}

constexpr int TC_ERR_GROUP_TIMEOUT = 3;                       // the error word's "grid barrier" code
constexpr unsigned long long TC_GROUP_TIMEOUT_NS = 20000000000ull;

// Barrier over the nct = gridDim.y CTAs of one group (co-resident: cooperative launch).  The group's 64-bit counter only
// ever grows: every CTA adds 1 per barrier, so barrier k of a launch completes at base + nct (k + 1), base being the counter
// before the launch (tc_group_init).  A value left by an earlier launch is <= base and never satisfies a wait.  The CTA
// barrier then the release-add order every thread's earlier stores before the arrival; the acquire poll then the CTA barrier
// order the peers' stores before every thread's later accesses.  Bounded by %globaltimer: a missing arrival raises the error
// word and turns this CTA's remaining waits into no-ops (target TC_GROUP_DEAD), so the kernel ends instead of hanging.
// The state lives in shared memory: nothing of it stays live in registers across the layers.
struct TcGroupBar {
    unsigned long long* ctr;      // the group's counter (end of its workspace slot)
    unsigned long long target;    // counter value that completes the next wait
};
constexpr unsigned long long TC_GROUP_DEAD = ~0ull;
__device__ __forceinline__ void tc_group_wait(TcGroupBar* gb, int* err_flag) {   // thread 0
    unsigned long long* ctr = gb->ctr;
    asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(ctr) : "memory");
    if (gb->target == TC_GROUP_DEAD) return;
    const unsigned long long target = gb->target + gridDim.y;
    gb->target = target;
    unsigned long long t0 = 0;
    for (unsigned spins = 1;; ++spins) {
        unsigned long long v;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ctr) : "memory");
        if (v >= target) return;
        if ((spins & 255u) == 0) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            if (t0 == 0) {
                t0 = t;
            } else if (t - t0 > TC_GROUP_TIMEOUT_NS) {
                if (err_flag) *reinterpret_cast<volatile int*>(err_flag) = TC_ERR_GROUP_TIMEOUT;
                __threadfence_system();
                gb->target = TC_GROUP_DEAD;
                return;
            }
        }
    }
}
__device__ __forceinline__ void tc_group_sync(TcGroupBar* gb, int* err_flag) {
    __syncthreads();
    if (threadIdx.x == 0) tc_group_wait(gb, err_flag);
    __syncthreads();
}
// The per-layer barrier: the CTA-level halves are over the 256 consumer threads only (the producer warp runs ahead into the
// next layer).  Thread 0 then hands the published X planes to the producer lane through the shared mbarrier `xpub` (one
// phase per layer barrier); the producer runs fence.proxy.async before its TMA reads them.  A dead group still arrives, so
// the producer is released.
__device__ __forceinline__ void tc_group_sync_consumers(TcGroupBar* gb, int* err_flag, uint64_t* xpub) {
    tc_consumer_sync();
    if (threadIdx.x == 0) {
        tc_group_wait(gb, err_flag);
        mbar_arrive(xpub);
    }
    tc_consumer_sync();
}
// Producer-warp wait on a hand-off that can lie behind a group barrier: backs off like mbar_wait_backoff, but is bounded by
// %globaltimer at twice the group-barrier timeout, so that a stalled peer ends the kernel through the barrier's error code
// (the barrier's own timeout always arrives first) rather than through this wait.
__device__ __forceinline__ void tc_wait_behind_group(uint64_t* bar, uint32_t parity, int* err_flag) {
    unsigned long long t0 = 0;
    for (unsigned spins = 1; !mbar_try_wait(bar, parity); ++spins) {
        __nanosleep(128);
        if ((spins & 255u) == 0) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            if (t0 == 0) {
                t0 = t;
            } else if (t - t0 > 2 * TC_GROUP_TIMEOUT_NS) {
                if (err_flag) *reinterpret_cast<volatile int*>(err_flag) = ERR_MBAR_TIMEOUT;
                __threadfence_system();
                __trap();
            }
        }
    }
}
// thread 0, before its first arrival: base = the counter before this launch.  Every earlier launch left it at a multiple of
// nct, and the peers of this launch can be at most nct - 1 arrivals past it (barrier 0 needs this CTA's arrival).
__device__ __forceinline__ void tc_group_init(TcGroupBar* gb, unsigned long long* ctr) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(ctr) : "memory");
    gb->ctr = ctr;
    gb->target = v - v % gridDim.y;
}

// float offset of element (row r, k) inside one [tile_rows x 16] plane
__device__ __forceinline__ size_t tc_plane_off(int r, int k_in_block, int tile_rows = TCM) {
    return (size_t)(k_in_block >> 2) * tile_rows * 4 + (size_t)(r >> 3) * 32 + (size_t)(r & 7) * 4 + (k_in_block & 3);
}

// W^T [Kpad][L] (the packed blob's layout) -> W planes [L/256][n_kb][hi|lo][256 x 16] with K padded to n_kb * 16
__global__ void tc_pack_weights_kernel(const float* __restrict__ wt, float* __restrict__ planes, int Kpad, int L, int n_kb) {
    const int K = n_kb * TCKB;
    const size_t plane = (size_t)TCN * TCKB;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)L * K; i += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(i / L), n = (int)(i % L);  // consecutive threads -> consecutive n: coalesced reads of W^T
        const float v = k < Kpad ? wt[(size_t)k * L + n] : 0.f;
        const float h = tc_tf32(v), l = tc_tf32(v - h);
        float* blk = planes + ((size_t)(n / TCN) * n_kb + k / TCKB) * 2 * plane;
        const size_t off = tc_plane_off(n % TCN, k % TCKB, TCN);
        blk[off] = h;
        blk[plane + off] = l;
    }
}

// profiling aid (mlb_debug_fwd_marks): CTA (0,0) stamps %globaltimer per layer of its first tile: thread 0 at [8g+0] layer start,
// [8g+3] accumulators complete, [8g+4] epilogue done, [8g+5] group barrier passed; MMA lane at [8g+1] first stage landed,
// [8g+2] all MMAs issued; producer lane at [8g+6] all stages issued, [8g+7] X copies of the layer issued (the X planes of
// layers g >= 1 wait for the group barrier of layer g-1; their W planes do not).  Per tile t < 4 of group 0, thread 0: [128+4t] tile
// start, [129+4t] prologue barrier passed, [130+4t] head partials gathered, [131+4t] rows stored.  Group barriers per tile:
// one after the prologue, one per layer (the last one also publishes the head partials).
__device__ unsigned long long* g_tc_marks = nullptr;
__device__ __forceinline__ void tmark(unsigned long long* marks, int slot) {
    if (marks != nullptr) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        marks[slot] = t;
    }
}

struct TcHeadGroups {     // the narrow heads' rows grouped by the GEMM layer that feeds them (g = 0, 1)
    int src[2];           // op index of the feeding layer (-1: no group)
    int q0[2], n[2];      // first head row, row count
    int nq[2], off[2];    // rows rounded up to 4, first hacc slot
};

struct TcEpi {            // what one epilogue pass over this thread's 64 columns needs
    const float* acc;     // shared: this thread's row of the staged accumulators (main + cross), at its first column
    const float* sst;     // shared: scale[256] | shift[256] of the CTA's columns
    const float* hw;      // shared: [NQ][256] weights of the head rows this layer feeds (zero rows beyond the real ones)
    float* nxt;           // next layer's X planes (cluster slot)
    float* res;           // fp32 residual [L/4][64][4] (cluster slot)
    int col0;             // first global column of the thread
    int ccol0;            // first CTA-local column of the thread (0, 64, 128 or 192)
    int tid, grow, site;
    bool live, relu, add_res, save_res, drop, write_planes;
    const uint8_t* drop_mask;
    int n_rows, L;
    uint32_t rm, thr;
    float inv_keep;
    uint64_t keep;        // L2 evict_last policy for the residual
};

// The fp32 residual of a stage is written two layers before it is read: ~110 MB of other L2 traffic pass in between and
// plain LRU had evicted it to HBM by then (100 MB of DRAM round trips per batch of 4096).  L2::evict_last keeps it resident.
__device__ __forceinline__ uint64_t tc_policy_evict_last() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void tc_st_keep(float* ptr, float4 v, uint64_t pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(ptr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ float4 tc_ld_keep(const float* ptr, uint64_t pol) {
    float4 v;
    asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(ptr), "l"(pol));
    return v;
}

// MC-dropout of four consecutive columns (rare path, kept out of line: the epilogue loops must stay small enough for the
// instruction cache -- fully unrolled they were 140 KB per instantiation and every first use cost ~15 us of code fetch)
__device__ __noinline__ float4 tc_dropout4(float4 v, const uint8_t* mask_row, uint32_t rm, uint32_t thr, float inv_keep, int gc, int site,
                                           int live) {
    float o[4] = {v.x, v.y, v.z, v.w};
    if (mask_row != nullptr) {
        if (live) {
            const uint32_t mk = *reinterpret_cast<const uint32_t*>(mask_row + gc);
#pragma unroll
            for (int t = 0; t < 4; ++t) o[t] = ((mk >> (8 * t)) & 0xFFu) ? o[t] * inv_keep : 0.f;
        }
    } else {
#pragma unroll
        for (int t = 0; t < 4; ++t) o[t] = drop_keep(rm, drop_col_hash((uint32_t)(gc + t), (uint32_t)site), thr) ? o[t] * inv_keep : 0.f;
    }
    return make_float4(o[0], o[1], o[2], o[3]);
}

constexpr int TC_CW = 16;   // accumulator columns per epilogue chunk

// One 16-column chunk of this thread's row: BN affine / ReLU / dropout / residual, head partial sums, hi / lo planes out.
template <int NQ, int OFF, bool ADD>
__device__ __forceinline__ void tc_epilogue_chunk(const TcEpi& e, int ch, const float* acc, const float4* rr, float* hacc) {
    constexpr size_t plane = (size_t)TCM * TCKB;
#pragma unroll
    for (int j4 = 0; j4 < TC_CW / 4; ++j4) {
        const int lc = e.ccol0 + TC_CW * ch + 4 * j4;   // CTA-local column
        const int gc = e.col0 + TC_CW * ch + 4 * j4;    // global column = k index of the next layer
        const float4 sc = *reinterpret_cast<const float4*>(e.sst + lc);
        const float4 sh = *reinterpret_cast<const float4*>(e.sst + TCN + lc);
        float v[4];
        const float4 a = *reinterpret_cast<const float4*>(acc + 4 * j4);
        v[0] = fmaf(a.x, sc.x, sh.x);
        v[1] = fmaf(a.y, sc.y, sh.y);
        v[2] = fmaf(a.z, sc.z, sh.z);
        v[3] = fmaf(a.w, sc.w, sh.w);
        if (e.relu) {
#pragma unroll
            for (int t = 0; t < 4; ++t) v[t] = fmaxf(v[t], 0.f);
        }
        if (e.drop) {
            const uint8_t* mrow = e.drop_mask ? e.drop_mask + ((size_t)e.site * e.n_rows + e.grow) * e.L : nullptr;
            const float4 d = tc_dropout4(make_float4(v[0], v[1], v[2], v[3]), mrow, e.rm, e.thr, e.inv_keep, gc, e.site, (int)e.live);
            v[0] = d.x, v[1] = d.y, v[2] = d.z, v[3] = d.w;
        }
        float* rq = e.res + ((size_t)(gc >> 2) * TCM + e.tid) * 4;   // a warp touches 512 contiguous bytes
        if (ADD) {
            const float4 r = rr[j4];
            v[0] += r.x, v[1] += r.y, v[2] += r.z, v[3] += r.w;
        }
        if (e.save_res) tc_st_keep(rq, make_float4(v[0], v[1], v[2], v[3]), e.keep);
#pragma unroll
        for (int q = 0; q < NQ; ++q) {   // narrow heads on this layer's output: partial dot products over my columns
            const float4 w = *reinterpret_cast<const float4*>(e.hw + q * TCN + lc);
            hacc[OFF + q] = fmaf(v[3], w.w, fmaf(v[2], w.z, fmaf(v[1], w.y, fmaf(v[0], w.x, hacc[OFF + q]))));
        }
        if (e.write_planes) {   // the last layer's output only feeds the heads
            float* blk = e.nxt + (size_t)(gc / TCKB) * 2 * plane;
            const float4 h = make_float4(tc_tf32(v[0]), tc_tf32(v[1]), tc_tf32(v[2]), tc_tf32(v[3]));
            const float4 l = make_float4(tc_tf32(v[0] - h.x), tc_tf32(v[1] - h.y), tc_tf32(v[2] - h.z), tc_tf32(v[3] - h.w));
            const size_t off = tc_plane_off(e.tid, gc % TCKB);
            *reinterpret_cast<float4*>(blk + off) = h;
            *reinterpret_cast<float4*>(blk + plane + off) = l;
        }
    }
}

// The 64 staged accumulator columns of this thread's row, 16 per (rolled) loop trip; the residual of the next chunk is in
// flight while the current one is processed.
template <int NQ, int OFF, bool ADD>
__device__ __forceinline__ void tc_epilogue_cols(const TcEpi& e, float* hacc) {
    constexpr int NCH = TCH / TC_CW, RW = ADD ? TC_CW / 4 : 1;
    const float* res_row = e.res + ((size_t)(e.col0 >> 2) * TCM + e.tid) * 4;   // + 256 floats per 4 columns
    float4 rr[RW], rn[RW];
    auto fetch = [&](int ch, float4* r) {
        if (ADD) {
#pragma unroll
            for (int j4 = 0; j4 < TC_CW / 4; ++j4) r[j4] = tc_ld_keep(res_row + (size_t)(ch * (TC_CW / 4) + j4) * TCM * 4, e.keep);
        }
    };
    fetch(0, rr);
#pragma unroll 1
    for (int ch = 0; ch < NCH; ++ch) {
        if (ch + 1 < NCH) fetch(ch + 1, rn);
        tc_epilogue_chunk<NQ, OFF, ADD>(e, ch, e.acc + TC_CW * ch, rr, hacc);
#pragma unroll
        for (int j = 0; j < RW; ++j) rr[j] = rn[j];
    }
}

template <bool IMAGES>
__global__ void __launch_bounds__(TC_THREADS, 1) loco_forward_tc_kernel(const __grid_constant__ FwdParams p,
                                                                        const __grid_constant__ TcExtra ex,
                                                                        const __grid_constant__ ImgParams ib) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // full[s]: two arrivals per fill (the W planes as soon as the slot is empty, the X planes once they are published);
    // empty[s]: one arrival per consumer warp.  cready / cfree[b]: epilogue-constant buffer b staged / read.  xpub: the
    // X planes of the next layer are published (thread 0, after the group barrier) -> the producer lane.
    __shared__ __align__(8) uint64_t full[TCNST], empty[TCNST], cready[2], cfree[2], xpub;
    __shared__ TcGroupBar gbar;
    __shared__ TcHeadGroups hgrp;   // kept in shared memory, out of the registers of the MMA loop
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nt = blockIdx.y, nct = gridDim.y, L = p.L;
    const bool epi_thread = tid < TC_EPI, prod_warp = tid >= TC_EPI, prod_lane = tid == TC_EPI;
    const int wg = (tid >> 7) & 1;     // consumer warpgroup: output columns [128 wg, 128 wg + 128) of the CTA's 256
    const int quarter = (tid >> 6) & 3;   // epilogue threads: which 64 columns of the CTA's 256 (quarters 2 wg, 2 wg + 1)
    // two buffers of epilogue constants, each scale | shift [2][256] then head weights [TC_HW][256]: layer g's buffer is
    // refilled at layer g+2, so the producer lane's copies never wait on the epilogue that reads the other one
    float* cbuf = reinterpret_cast<float*>(smem_raw + TC_RING_BYTES);
    float* hpart = reinterpret_cast<float*>(smem_raw);   // [4 nct][64][TC_HW] on CTA 0; aliases the idle ring

    // this group's workspace slot
    int first_gemm = 0;
    while (p.ops[first_gemm].type != MLB_OP_GEMM) ++first_gemm;
    const int n_kb0 = ex.n_kb[first_gemm];
    const size_t plane = (size_t)TCM * TCKB;
    float* slot = ex.ws + (size_t)blockIdx.x * ex.slot_floats;
    float* xin = slot;                                   // [n_kb0][hi|lo][64 x 16]
    float* xpl[2] = {xin + (size_t)n_kb0 * 2 * plane, xin + (size_t)n_kb0 * 2 * plane + (size_t)(L / TCKB) * 2 * plane};
    float* res = xpl[1] + (size_t)(L / TCKB) * 2 * plane;  // [L/4][64][4] fp32

    if (tid == 0) {
        // every consumer warp releases a stage once its warpgroup's wgmma reading it have retired
        for (int s = 0; s < TCNST; ++s) mbar_init(&full[s], 2), mbar_init(&empty[s], TC_EPI / 32);
        // cready: the producer lane's bulk copies (expect_tx) + the 31 other producer lanes' zero rows
        for (int b = 0; b < 2; ++b) mbar_init(&cready[b], 32), mbar_init(&cfree[b], TC_EPI / 32);
        mbar_init(&xpub, 1);
        mbar_fence_init();
        // after the residual: [4 nct][64][TC_HW] head partials of every CTA of the group, then the barrier counter
        tc_group_init(&gbar, reinterpret_cast<unsigned long long*>(res + (size_t)TCM * L + (size_t)4 * nct * TCM * TC_HW));
        // head rows are grouped by the layer that feeds them (at most two groups: w_aux | w_fin, or MonolocoModel.w2);
        // group g accumulates into hacc[off_g .. off_g + nq_g), nq_g = its row count rounded up to 4 (zero weights
        // beyond the real rows)
        int src[2] = {-1, -1}, q0[2] = {0, 0}, n[2] = {0, 0};
        for (int q = 0; q < ex.n_head_rows; ++q) {
            const int g = (src[0] < 0 || src[0] == ex.head_src[q]) ? 0 : 1;
            if (n[g] == 0) src[g] = ex.head_src[q], q0[g] = q;
            n[g]++;
        }
        for (int g = 0; g < 2; ++g) hgrp.src[g] = src[g], hgrp.q0[g] = q0[g], hgrp.n[g] = n[g], hgrp.nq[g] = (n[g] + 3) & ~3;
        hgrp.off[0] = 0, hgrp.off[1] = hgrp.nq[0];
    }
    __syncthreads();
    const int* grp_src = hgrp.src;
    const int* grp_q0 = hgrp.q0;
    const int* grp_n = hgrp.n;
    const int* grp_nq = hgrp.nq;
    const int* grp_off = hgrp.off;

    const float zm = p.z_met;
    const float k0 = p.kinv[0], k1 = p.kinv[1], k2 = p.kinv[2], k3 = p.kinv[3], k4 = p.kinv[4], k5 = p.kinv[5];
    const bool mc_drop = (p.flags & MLB_FWD_DROPOUT) != 0;
    int n_gemm = 0;
    for (int oi = 0; oi < p.n_ops; ++oi) n_gemm += p.ops[oi].type == MLB_OP_GEMM;

    unsigned long long* marks = (blockIdx.x == 0 && blockIdx.y == 0 && (tid == 0 || prod_lane)) ? g_tc_marks : nullptr;
    // ring stages and GEMM layers of the layers before this thread's current one (the producer warp is ahead of the
    // consumers, each counts its own): stage it uses slot it % TCNST, layer n uses constant buffer n & 1
    unsigned it0 = 0, n_lay = 0;
    float acc_m[TCWN / 2], acc_c[TCWN / 2];   // this thread's wgmma fragments: main (a_hi.w_hi) and cross terms
    for (int rb = (int)blockIdx.x; rb < ex.n_tiles; rb += (int)gridDim.x) {
        unsigned long long* tmk = (tid == 0 && rb < 4 * (int)gridDim.x) ? marks : nullptr;   // group 0's first four tiles
        const int tslot = 128 + 4 * (rb / (int)gridDim.x);
        tmark(tmk, tslot);
        const int row = tid & (TCM - 1);      // epilogue threads: my row of the tile
        const int grow = rb * TCM + row;      // my detection
        const bool live = epi_thread && grow < p.n_rows;
        const bool row_owner = epi_thread && quarter == 0;   // one thread per row does the prologue / the final store
        float cenrow[4] = {0.f, 0.f, 0.f, 0.f};

        // ------------------------------------------------------------ prologue: network input of my row -> hi / lo planes
        // every CTA of the group evaluates its row (cheap); CTA nt writes k blocks nt, nt + nct, ...
        if (row_owner) {
            float xr[KIN_MAX + 8];
#pragma unroll
            for (int k = 0; k < KIN_MAX + 8; ++k) xr[k] = 0.f;
            if (live) {
                if (p.input_kind == MLB_IN_X) {
#pragma unroll
                    for (int k = 0; k < KIN_MAX; ++k)
                        if (k < p.in_size) xr[k] = __ldg(p.x + (size_t)grow * p.in_size + k);
                } else if constexpr (IMAGES) {
                    // the row's own K^-1 and poses (fwd_common.cuh)
                    preprocess_row_images(p, ib, grow, true, cenrow, [&](int k, float v) { xr[k] = v; });
                } else {
                    const bool stereo = p.input_kind == MLB_IN_KPS_STEREO;
                    const float* kp = p.x + (size_t)(stereo ? grow / p.n_right : grow) * 51;
                    const float* kr = stereo ? p.xr + (size_t)(grow % p.n_right) * 51 : nullptr;
                    float umin = __ldg(kp), umax = umin, vmin = __ldg(kp + 17), vmax = vmin;
                    for (int j = 1; j < 17; ++j) {
                        const float u = __ldg(kp + j), v = __ldg(kp + 17 + j);
                        umin = fminf(umin, u), umax = fmaxf(umax, u);
                        vmin = fminf(vmin, v), vmax = fmaxf(vmax, v);
                    }
                    const float uc = __fadd_rn(__fdiv_rn(__fsub_rn(umax, umin), 2.f), umin);  // camera.py:82-86
                    const float vc = __fadd_rn(__fdiv_rn(__fsub_rn(vmax, vmin), 2.f), vmin);
                    cenrow[0] = uc, cenrow[1] = vc;
                    cenrow[2] = (uc * k0 + vc * k1 + k2) * zm;
                    cenrow[3] = (uc * k3 + vc * k4 + k5) * zm;
                    const bool zc = (p.flags & MLB_FWD_ZERO_CENTER) != 0;
#pragma unroll
                    for (int j = 0; j < 17; ++j) {
                        const float u = __ldg(kp + j), v = __ldg(kp + 17 + j);
                        float xl = (u * k0 + v * k1 + k2) * zm;  // camera.py:26-27, rows 0/1 of [u v 1] K^-T
                        float yl = (u * k3 + v * k4 + k5) * zm;
                        if (stereo) {
                            const float ur = __ldg(kr + j), vr = __ldg(kr + 17 + j);
                            xr[34 + 2 * j] = xl - (ur * k0 + vr * k1 + k2) * zm;  // process.py:41 cat(l, l - r)
                            xr[35 + 2 * j] = yl - (ur * k3 + vr * k4 + k5) * zm;
                        } else if (zc) {
                            xl -= cenrow[2];  // process.py:61-62
                            yl -= cenrow[3];
                        }
                        xr[2 * j] = xl, xr[2 * j + 1] = yl;
                    }
                }
                if (nt == 0 && p.out_x != nullptr && p.input_kind != MLB_IN_X) {
#pragma unroll
                    for (int k = 0; k < KIN_MAX; ++k)
                        if (k < p.in_size) p.out_x[(size_t)grow * p.in_size + k] = xr[k];
                }
            }
#pragma unroll
            for (int kb = 0; kb < (KIN_MAX + 8) / TCKB; ++kb) {
                if (kb < n_kb0 && (kb % nct) == nt) {
                    float* blk = xin + (size_t)kb * 2 * plane;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float4 v = make_float4(xr[kb * 16 + 4 * q], xr[kb * 16 + 4 * q + 1], xr[kb * 16 + 4 * q + 2], xr[kb * 16 + 4 * q + 3]);
                        const float4 h = make_float4(tc_tf32(v.x), tc_tf32(v.y), tc_tf32(v.z), tc_tf32(v.w));
                        const float4 l = make_float4(tc_tf32(v.x - h.x), tc_tf32(v.y - h.y), tc_tf32(v.z - h.z), tc_tf32(v.w - h.w));
                        const size_t off = tc_plane_off(row, 4 * q);
                        *reinterpret_cast<float4*>(blk + off) = h;
                        *reinterpret_cast<float4*>(blk + plane + off) = l;
                    }
                }
            }
        }
        tc_group_sync(&gbar, p.err_flag);   // the input planes of this tile are complete (and the previous tile's tail
                                            // is over everywhere)
        tmark(tmk, tslot + 1);

        int par = 0, site = 0, gi = 0;  // gi: GEMM ops done in this tile
        for (int oi = 0; oi < p.n_ops; ++oi) {
            const mlb_op& op = p.ops[oi];
            if (op.type != MLB_OP_GEMM) continue;
            const int n_kb = ex.n_kb[oi];
            // this layer's X planes and head group (-1: none), evaluated where used: neither stays live across the MMAs
            auto x_src = [&]() { return reinterpret_cast<const unsigned char*>(gi == 0 ? xin : xpl[par]); };
            auto head_group = [&]() { return grp_src[0] == oi ? 0 : (grp_src[1] == oi ? 1 : -1); };
            unsigned long long* mk = (rb == 0 && gi < 15) ? marks : nullptr;
            if (tid == 0) tmark(mk, 8 * gi + 0);
            auto const_buf = [&](unsigned n) { return cbuf + (size_t)(n & 1) * (TC_CONST_BYTES / sizeof(float)); };

            if (prod_lane) {
                // ---- producer: this row tile's X planes and this column tile's W planes, 40 KB per stage.  Within a tile
                // this lane runs ahead of the consumers: the W planes of a layer's first stages do not depend on the
                // activations, so they stream while the previous layer's last MMAs, epilogue and group barrier run (its
                // staging tile sits in the other two slots); the X planes follow once thread 0 hands them over (xpub).
                const unsigned char* xsrc = x_src();
                const unsigned char* wsrc = reinterpret_cast<const unsigned char*>(ex.wplanes[oi]) + (size_t)nt * n_kb * 2 * TC_W_PLANE;
                auto fill_w = [&](int kb) {
                    const unsigned it = it0 + kb, s = it % TCNST;
                    if (it >= TCNST) mbar_wait(&empty[s], ((it / TCNST) - 1) & 1, p.err_flag);
                    mbar_expect_tx(&full[s], 2 * TC_W_PLANE);
                    tma_bulk_g2s(smem_raw + (size_t)s * TC_STAGE + 2 * TC_A_PLANE, wsrc + (size_t)kb * 2 * TC_W_PLANE, 2 * TC_W_PLANE, &full[s]);
                };
                auto fill_x = [&](int kb) {   // after fill_w(kb): the slot is empty
                    const unsigned s = (it0 + kb) % TCNST;
                    mbar_expect_tx(&full[s], 2 * TC_A_PLANE);
                    tma_bulk_g2s(smem_raw + (size_t)s * TC_STAGE, xsrc + (size_t)kb * 2 * TC_A_PLANE, 2 * TC_A_PLANE, &full[s]);
                };
                int kb = 0;
                if (gi > 0)
                    for (; kb < n_kb && kb < TCNST; ++kb) fill_w(kb);
                // xpub: one phase per layer barrier (layer 0 of a tile follows the CTA-wide prologue barrier, which is
                // later than the previous tile's last phase)
                if (n_lay > 0) tc_wait_behind_group(&xpub, (n_lay - 1) & 1, p.err_flag);
                // the prologue barrier (layer 0) or xpub ordered the peers' generic-proxy stores (planes, hpart) before
                // this point: -> async-proxy TMA
                asm volatile("fence.proxy.async;" ::: "memory");
                for (int k = 0; k < kb; ++k) fill_x(k);
                if (kb == 0) fill_w(0), fill_x(0), kb = 1;
                tmark(mk, 8 * gi + 7);
                {
                    // this layer's epilogue constants, as bulk copies into buffer n_lay & 1 (every blob array is 128-byte
                    // aligned): folded-BN scale | shift and the real rows of the head group fed here.  Issued here, the
                    // copies neither delay the layer's first X copies nor stall this lane behind global loads.
                    const unsigned b = n_lay & 1;
                    float* sst = const_buf(n_lay);
                    const int hg = head_group();
                    const int nrow = hg >= 0 ? grp_n[hg] : 0;
                    if (n_lay >= 2) mbar_wait(&cfree[b], ((n_lay >> 1) - 1) & 1, p.err_flag);
                    mbar_expect_tx(&cready[b], (uint32_t)(2 + nrow) * TCN * sizeof(float));
                    tma_bulk_g2s(sst, p.blob + op.scale_off + nt * TCN, TCN * sizeof(float), &cready[b]);
                    tma_bulk_g2s(sst + TCN, p.blob + op.shift_off + nt * TCN, TCN * sizeof(float), &cready[b]);
                    for (int r = 0; r < nrow; ++r)
                        tma_bulk_g2s(sst + (2 + r) * TCN, p.blob + ex.head_w[grp_q0[hg] + r] + nt * TCN, TCN * sizeof(float), &cready[b]);
                }
                for (; kb < n_kb; ++kb) fill_w(kb), fill_x(kb);
                tmark(mk, 8 * gi + 6);
            } else if (prod_warp) {
                // ---- the other producer lanes: zero head-weight rows beyond the real ones (rows rounded up to 4) in this
                // layer's constant buffer, once the epilogue two layers back has read it.  Stores only: global loads on
                // these lanes stalled the producer lane that shares their warp (its first copies by up to 28 us, or
                // the MMA stream, in tools/tc_marks.py), so the constants themselves come by bulk copy.
                float* hw = const_buf(n_lay) + 2 * TCN;   // [TC_HW][256]
                const int hg = head_group();
                if (n_lay >= 2) tc_wait_behind_group(&cfree[n_lay & 1], ((n_lay >> 1) - 1) & 1, p.err_flag);
                if (hg >= 0)
                    for (int i = grp_n[hg] * TCN + lane - 1; i < grp_nq[hg] * TCN; i += 31) hw[i] = 0.f;
                mbar_arrive(&cready[n_lay & 1]);
            } else {
                // ---- consumer warpgroup wg: 2 k-steps x 3 wgmma (M 64, N 128, K 8) per stage, one stage in flight
#pragma unroll
                for (int i = 0; i < TCWN / 2; ++i) acc_m[i] = 0.f, acc_c[i] = 0.f;
                for (int kb = 0; kb < n_kb; ++kb) {
                    const unsigned it = it0 + kb, s = it % TCNST;
                    mbar_wait(&full[s], (it / TCNST) & 1, p.err_flag);
                    if (kb == 0 && tid == 0) tmark(mk, 8 * gi + 1);
                    const uint32_t a_hi = smem_u32(smem_raw + (size_t)s * TC_STAGE), a_lo = a_hi + TC_A_PLANE;
                    const uint32_t w_hi = a_hi + 2 * TC_A_PLANE + (uint32_t)wg * (TCWN / 8) * TC_SBO, w_lo = w_hi + TC_W_PLANE;
                    tc_wgmma_fence();
#pragma unroll
                    for (int j = 0; j < TCKB / 8; ++j) {
                        const uint64_t ah = tc_desc(a_hi + 2 * j * TC_LBO_A, TC_LBO_A), al = tc_desc(a_lo + 2 * j * TC_LBO_A, TC_LBO_A);
                        const uint64_t wh = tc_desc(w_hi + 2 * j * TC_LBO_W, TC_LBO_W), wl = tc_desc(w_lo + 2 * j * TC_LBO_W, TC_LBO_W);
                        tc_wgmma(acc_c, al, wh);
                        tc_wgmma(acc_c, ah, wl);
                        tc_wgmma(acc_m, ah, wh);
                    }
                    tc_wgmma_commit();
                    tc_wgmma_wait<1>();   // the previous stage's group has retired: release its slot
                    tc_fence_regs(acc_m), tc_fence_regs(acc_c);
                    // the layer's last two stages stay held: their slots take the staging tiles (released after the epilogue)
                    if (kb > 0 && kb + 1 < n_kb && lane == 0) mbar_arrive(&empty[(it - 1) % TCNST]);
                }
                tc_wgmma_wait<0>();
                tc_fence_regs(acc_m), tc_fence_regs(acc_c);
                if (tid == 0) tmark(mk, 8 * gi + 2);
                tc_consumer_sync();   // both warpgroups are done reading the ring: stage the accumulators over it
                // warpgroup wg stages its 64 x 128 summed accumulators into the slot of this layer's stage n - 2 + wg
                // (n = it0 + n_kb, n_kb >= 2), which is the next layer's stage n + 2 + wg: the producer fills that layer's
                // first two stages meanwhile.  The warpgroup's epilogue threads (quarters 2 wg, 2 wg + 1) read only this tile.
                float* stg = reinterpret_cast<float*>(smem_raw + (size_t)((it0 + n_kb + 2 + wg) % TCNST) * TC_STAGE);   // [64][TC_SLD]
                {
                    // fragment of wgmma m64nNk8: warp w of the warpgroup holds rows 16w .. 16w + 15; lane l rows
                    // 16w + l/4 (+ 8), columns 8g + 2 (l % 4) (+ 1) of every 8-column group g
                    const int r0 = 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
                    for (int g = 0; g < TCWN / 8; ++g) {
                        float* d = stg + (size_t)r0 * TC_SLD + c0 + 8 * g;
                        *reinterpret_cast<float2*>(d) = make_float2(acc_m[4 * g] + acc_c[4 * g], acc_m[4 * g + 1] + acc_c[4 * g + 1]);
                        *reinterpret_cast<float2*>(d + 8 * TC_SLD) =
                            make_float2(acc_m[4 * g + 2] + acc_c[4 * g + 2], acc_m[4 * g + 3] + acc_c[4 * g + 3]);
                    }
                }
            }
            if (epi_thread) {
                const float* stg = reinterpret_cast<const float*>(smem_raw + (size_t)((it0 + n_kb + 2 + wg) % TCNST) * TC_STAGE);
                tc_warpgroup_sync(wg);                                         // my warpgroup's staging tile is complete
                mbar_wait(&cready[n_lay & 1], (n_lay >> 1) & 1, p.err_flag);   // this layer's epilogue constants are staged
                const int hg = head_group();
                const bool head_layer = hg >= 0;
                TcEpi e;
                e.sst = const_buf(n_lay), e.hw = e.sst + 2 * TCN, e.nxt = xpl[gi == 0 ? 0 : (par ^ 1)], e.res = res;
                e.tid = row, e.grow = grow, e.site = site, e.live = live;
                e.relu = (op.flags & MLB_F_RELU) != 0, e.add_res = (op.flags & MLB_F_ADD_RES) != 0;
                e.save_res = (op.flags & MLB_F_SAVE_RES) != 0, e.drop = mc_drop && (op.flags & MLB_F_DROPOUT) != 0;
                e.write_planes = gi + 1 < n_gemm;
                e.drop_mask = p.drop_mask, e.n_rows = p.n_rows, e.L = L;
                e.rm = drop_row_mix(drop_seed_mix(p.drop_seed), (uint32_t)grow), e.thr = drop_threshold(p.p_drop);
                e.inv_keep = 1.0f / (1.0f - p.p_drop);
                e.keep = tc_policy_evict_last();
                if (tid == 0) tmark(mk, 8 * gi + 3);
                e.ccol0 = TCH * quarter, e.col0 = nt * TCN + TCH * quarter;
                e.acc = stg + (size_t)row * TC_SLD + TCH * (quarter & 1);
                float hacc[TC_HW];   // head partial sums over my 64 columns; slots [off, off + nq) of the group fed here
#pragma unroll
                for (int q = 0; q < TC_HW; ++q) hacc[q] = 0.f;
                if (!head_layer) {
                    if (e.add_res) tc_epilogue_cols<0, 0, true>(e, hacc);
                    else tc_epilogue_cols<0, 0, false>(e, hacc);
                } else if (e.add_res) {   // MonolocoModel: the last stage's output (x + y) feeds the only head
                    const int nqg = grp_nq[hg];
                    if (nqg <= 4) tc_epilogue_cols<4, 0, true>(e, hacc);
                    else if (nqg <= 8) tc_epilogue_cols<8, 0, true>(e, hacc);
                    else if (nqg <= 12) tc_epilogue_cols<12, 0, true>(e, hacc);
                    else tc_epilogue_cols<16, 0, true>(e, hacc);
                } else {   // (rows of this group rounded to 4, offset of the group)
                    const int nqg = grp_nq[hg], off = grp_off[hg];
                    if (off == 0) {
                        if (nqg <= 4) tc_epilogue_cols<4, 0, false>(e, hacc);
                        else if (nqg <= 8) tc_epilogue_cols<8, 0, false>(e, hacc);
                        else if (nqg <= 12) tc_epilogue_cols<12, 0, false>(e, hacc);
                        else tc_epilogue_cols<16, 0, false>(e, hacc);
                    } else if (off == 4) {
                        if (nqg <= 4) tc_epilogue_cols<4, 4, false>(e, hacc);
                        else if (nqg <= 8) tc_epilogue_cols<8, 4, false>(e, hacc);
                        else tc_epilogue_cols<12, 4, false>(e, hacc);
                    } else if (off == 8) {
                        if (nqg <= 4) tc_epilogue_cols<4, 8, false>(e, hacc);
                        else tc_epilogue_cols<8, 8, false>(e, hacc);
                    } else {
                        tc_epilogue_cols<4, 12, false>(e, hacc);
                    }
                }
                if (head_layer) {   // -> the group slot, [4 nt + quarter][row][TC_HW]; CTA 0 sums them after the last layer
                    const int q4a = grp_off[hg] / 4, q4b = (grp_off[hg] + grp_nq[hg]) / 4;
                    float4* dst = reinterpret_cast<float4*>(res + (size_t)TCM * L + ((size_t)(4 * nt + quarter) * TCM + row) * TC_HW);
#pragma unroll
                    for (int q4 = 0; q4 < TC_HW / 4; ++q4)
                        if (q4 >= q4a && q4 < q4b) dst[q4] = make_float4(hacc[4 * q4], hacc[4 * q4 + 1], hacc[4 * q4 + 2], hacc[4 * q4 + 3]);
                }
                // the staging tile and the constants are read: the two held slots go back to the producer lane (this
                // thread's generic-proxy accesses ordered before its async-proxy refills) and the constant buffer to the
                // other producer lanes
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(&empty[(it0 + n_kb - 2) % TCNST]);
                    mbar_arrive(&empty[(it0 + n_kb - 1) % TCNST]);
                    mbar_arrive(&cfree[n_lay & 1]);
                }
                if (tid == 0) tmark(mk, 8 * gi + 4);
                // all column tiles of this row tile are written; then the X planes of the next layer go to the producer
                tc_group_sync_consumers(&gbar, p.err_flag, &xpub);
                if (tid == 0) tmark(mk, 8 * gi + 5);
                // The planes this layer read are dead now (every CTA of the group is past its MMAs) and will be fully
                // rewritten before their next use: drop the dirty lines from L2 instead of letting them be written back to
                // HBM (discard.global.L2; without it the workspace churn was 255 MB of DRAM writes per batch of 4096).
                const size_t lines = (size_t)n_kb * 2 * TC_A_PLANE / 128;   // 128-byte lines; CTA nt takes lines nt, nt + nct, ...
                const unsigned char* base = x_src();
                for (size_t ln = (size_t)nt + (size_t)nct * tid; ln < lines; ln += (size_t)nct * TC_EPI)
                    asm volatile("discard.global.L2 [%0], 128;" ::"l"(base + ln * 128) : "memory");
                if ((op.flags & MLB_F_ADD_RES) && !(op.flags & MLB_F_SAVE_RES)) {   // last use of the stage residual
                    const unsigned char* rb = reinterpret_cast<const unsigned char*>(res + (size_t)(nt * TCN / 4) * TCM * 4);
                    for (size_t o = (size_t)tid * 128; o < (size_t)TCN * TCM * 4; o += (size_t)TC_EPI * 128)
                        asm volatile("discard.global.L2 [%0], 128;" ::"l"(rb + o) : "memory");
                }
            }
            if (op.flags & MLB_F_DROPOUT) site++;
            if (gi > 0) par ^= 1;
            ++gi, ++n_lay, it0 += n_kb;
        }
        // the producer warp rejoins: the tail aliases the ring (hpart) and the constants (gather staging), and the last
        // layer's group barrier ordered the peers' head partials before this point
        __syncwarp();
        __syncthreads();

        // ------------------------------------------------------------ tail: head partials (slot) -> CTA 0 -> decode + stores
        // the head layers wrote every CTA's partials to the slot; the last layer's group barrier ordered them before this point
        if (nt == 0) {
            // all partials into shared memory (the ring is idle) with independent 16-byte loads, then the fixed-order sum
            const float4* src = reinterpret_cast<const float4*>(res + (size_t)TCM * L);   // [4 nct][64][TC_HW]
            float4* dst = reinterpret_cast<float4*>(hpart);
            for (int i = tid; i < nct * TCM * TC_HW; i += TC_THREADS) dst[i] = __ldcg(src + i);   // 4 nct x 64 x 16 floats
            __syncthreads();
            tmark(tmk, tslot + 2);
        }
        if (nt == 0 && live && row_owner) {
            float o[OUT_LD];
#pragma unroll
            for (int k = 0; k < OUT_LD; ++k) o[k] = 0.f;
            for (int q = 0; q < ex.n_head_rows; ++q) {
                const int g = (q >= grp_q0[1] && grp_n[1] > 0) ? 1 : 0;
                const int slot = grp_off[g] + (q - grp_q0[g]);
                float s = 0.f;
                for (int t = 0; t < 4 * nct; ++t) s += hpart[((size_t)t * TCM + row) * TC_HW + slot];  // fixed order: deterministic
                o[ex.head_col[q]] = s + __ldg(p.blob + ex.head_b[q]);
            }
            store_row<IMAGES>(p, (size_t)grow, o, cenrow, p.n_gather ? cbuf + (size_t)row * MLB_GATHER_LD : nullptr, &ib);
        }
        if (nt == 0 && p.n_gather) {
            // fused all-gather: the tile's rows ([<=64][20] floats, contiguous in every gather buffer) leave as coalesced
            // 16-byte stores -- 128-byte NVLink packets instead of 11 scattered 4..16-byte stores per row and peer
            // (the constant buffers are free here: the tile's layers are done; the next tile stages them after its
            // prologue barrier)
            __syncthreads();
            const int rows_live = min(TCM, p.n_rows - rb * TCM);
            const int n4 = rows_live * (MLB_GATHER_LD / 4);
            const float4* src = reinterpret_cast<const float4*>(cbuf);
            for (int pg = 0; pg < p.n_gather; ++pg) {
                float4* dst = reinterpret_cast<float4*>(p.gather[pg] + (size_t)(p.gather_row0 + (long long)rb * TCM) * MLB_GATHER_LD);
                for (int i = tid; i < n4; i += TC_THREADS) dst[i] = src[i];
            }
            __syncthreads();   // peer stores ordered before this CTA's arrival in gather_finish() (barrier + its fence)
        }
        tmark(tmk, tslot + 3);
        // the next tile's prologue ends with a group barrier: CTA 0 has copied the partials before any peer writes them
        // again, and has read its shared copy before its own producer refills the ring it aliases (program order +
        // fence.proxy.async)
    }
    if (nt == 0) {
        __syncthreads();  // every storing thread has fenced its peer stores (store_row)
        if (tid == 0) gather_finish(p);  // fused all-gather: one arrival per group leader
    }
}

}  // namespace mlb

// ================================================================================================ host side
using namespace mlb;

cudaError_t mlb_tc_set_marks(unsigned long long* ptr) { return cudaMemcpyToSymbol(mlb::g_tc_marks, &ptr, sizeof(ptr)); }

struct mlb_tc_state {
    float* wplanes[MLB_MAX_OPS];
    int n_kb[MLB_MAX_OPS];
    float* ws;
    size_t slot_floats;
    int max_groups;
    int nct;     // CTAs per group = L / 256
};

// widths the tensor-core kernel covers: 256 output columns per CTA, groups of up to 8 CTAs
bool mlb_tc_supported(int L) { return L >= TCN && L % TCN == 0 && L / TCN <= TC_MAX_CT; }

// pack the weight planes, size the workspace (one slot per co-resident group).  Returns nullptr + *err on failure.
mlb_tc_state* mlb_tc_prepare(const float* blob_dev, const mlb_op* ops, int n_ops, int L, cudaStream_t st, cudaError_t* err) {
    mlb_tc_state* t = new mlb_tc_state();
    memset(t, 0, sizeof(*t));
    t->nct = L / TCN;
    *err = cudaFuncSetAttribute(loco_forward_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM_BYTES);
    if (*err == cudaSuccess)
        *err = cudaFuncSetAttribute(loco_forward_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC_SMEM_BYTES);
    if (*err != cudaSuccess) { delete t; return nullptr; }
    int first = -1;
    for (int i = 0; i < n_ops; ++i) {
        if (ops[i].type != MLB_OP_GEMM) continue;
        if (first < 0) first = i;
        t->n_kb[i] = (ops[i].Kpad + TCKB - 1) / TCKB;
        // at least two k blocks (zero-padded): a layer's last two ring slots take the accumulator staging tiles
        if (t->n_kb[i] < 2) t->n_kb[i] = 2;
        const size_t fl = (size_t)2 * t->n_kb[i] * TCKB * L;
        if ((*err = cudaMalloc(&t->wplanes[i], fl * sizeof(float))) != cudaSuccess) return nullptr;
        tc_pack_weights_kernel<<<264, 256, 0, st>>>(blob_dev + ops[i].w_off, t->wplanes[i], ops[i].Kpad, L, t->n_kb[i]);
    }
    // groups: as many as the co-resident CTAs hold (the cooperative launch needs all of them resident at once)
    int dev = 0, sms = 0, per_sm = 0;
    if ((*err = cudaGetDevice(&dev)) != cudaSuccess) return nullptr;
    if ((*err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return nullptr;
    if ((*err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, loco_forward_tc_kernel<false>, TC_THREADS, TC_SMEM_BYTES)) != cudaSuccess)
        return nullptr;
    int n = per_sm * sms / t->nct;
    if (n < 1) {
        *err = cudaErrorCooperativeLaunchTooLarge;
        return nullptr;
    }
    if (getenv("MLB_TC_CLUSTERS") && atoi(getenv("MLB_TC_CLUSTERS")) > 0 && atoi(getenv("MLB_TC_CLUSTERS")) < n) n = atoi(getenv("MLB_TC_CLUSTERS"));
    t->max_groups = n;
    // slot: input planes, two plane sets, the fp32 residual, the head partials, the barrier counter (own 128-byte line)
    const size_t plane = (size_t)TCM * TCKB;
    t->slot_floats = (size_t)t->n_kb[first] * 2 * plane + 2 * (size_t)(L / TCKB) * 2 * plane + (size_t)TCM * L +
                     (size_t)4 * t->nct * TCM * TC_HW + 32;
    if ((*err = cudaMalloc(&t->ws, (size_t)n * t->slot_floats * sizeof(float))) != cudaSuccess) return nullptr;
    if ((*err = cudaMemsetAsync(t->ws, 0, (size_t)n * t->slot_floats * sizeof(float), st)) != cudaSuccess) return nullptr;
    *err = cudaGetLastError();
    return t;
}

cudaError_t mlb_tc_repack(mlb_tc_state* t, const float* blob_dev, const mlb_op* ops, int n_ops, int L, cudaStream_t st) {
    for (int i = 0; i < n_ops; ++i)
        if (ops[i].type == MLB_OP_GEMM)
            tc_pack_weights_kernel<<<264, 256, 0, st>>>(blob_dev + ops[i].w_off, t->wplanes[i], ops[i].Kpad, L, t->n_kb[i]);
    return cudaGetLastError();
}

void mlb_tc_free(mlb_tc_state* t) {
    if (!t) return;
    for (int i = 0; i < MLB_MAX_OPS; ++i) cudaFree(t->wplanes[i]);
    cudaFree(t->ws);
    delete t;
}

int mlb_tc_groups(const mlb_tc_state* t, int n_rows) {
    const int tiles = (n_rows + TCM - 1) / TCM;
    return tiles < t->max_groups ? tiles : t->max_groups;
}
int mlb_tc_max_groups(const mlb_tc_state* t) { return t->max_groups; }
int mlb_tc_tile_rows() { return TCM; }

cudaError_t mlb_tc_launch(const mlb_tc_state* t, const FwdParams& p, const ImgParams* ib, cudaStream_t st) {
    TcExtra ex;
    memset(&ex, 0, sizeof(ex));
    for (int i = 0; i < MLB_MAX_OPS; ++i) ex.wplanes[i] = t->wplanes[i], ex.n_kb[i] = t->n_kb[i];
    ex.ws = t->ws, ex.slot_floats = t->slot_floats;
    ex.n_tiles = (p.n_rows + TCM - 1) / TCM;
    int last_gemm = -1;
    for (int i = 0; i < p.n_ops; ++i) {
        const mlb_op& op = p.ops[i];
        if (op.type == MLB_OP_GEMM) {
            last_gemm = i;
        } else {
            if (last_gemm < 0) return cudaErrorInvalidValue;
            for (int o = 0; o < op.N; ++o) {
                if (ex.n_head_rows >= TC_HW) return cudaErrorInvalidValue;
                const int q = ex.n_head_rows++;
                ex.head_src[q] = last_gemm, ex.head_col[q] = op.out_col + o;
                ex.head_w[q] = op.w_off + (long long)o * op.K, ex.head_b[q] = op.shift_off + o;
            }
        }
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(mlb_tc_groups(t, p.n_rows), t->nct);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = TC_SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute at;
    at.id = cudaLaunchAttributeCooperative;   // co-residency: the CTAs of a group spin on each other's arrivals
    at.val.cooperative = 1;
    cfg.attrs = &at, cfg.numAttrs = 1;
    // the multi-image instantiation has the same shared memory and register budget (__launch_bounds__), so the same
    // per-SM occupancy and group count
    if (ib) return cudaLaunchKernelEx(&cfg, loco_forward_tc_kernel<true>, p, ex, *ib);
    return cudaLaunchKernelEx(&cfg, loco_forward_tc_kernel<false>, p, ex, ImgParams{});
}
