// kintinuous_b200 -- projective point-to-plane ICP: per-pixel residual / Jacobian row and the
// 6x6 [J^T J | J^T r] reduction, with the Gauss-Newton solve fused into the reduction's tail.
//
// Replaces (reference, src/frontend/):
//   icpStep + ICPReduction::search/getProducts + icpKernel + reduceSum   cuda/reduce.cu:186-419
//   struct JtJJtrSE3 (29 floats)                                         cuda/internal.h:98-149
//   the host half of ICPOdometry::getIncrementalTransformation           ICPOdometry.cpp:86-180
//
// Design (DESIGN.md section 3.2): the reference launches 64 CTAs x 128 threads (8 192 threads on a 132-SM part), a second
// 1-CTA kernel, then cudaDeviceSynchronize + 116-byte D2H + host LDLT, 19x per frame.  Two kernels here:
//   icp_frame_kernel  the tracker's path: ONE persistent cooperative launch per FRAME (132 CTAs x 512 threads, one per SM) runs all
//                     levels and iterations; the CTA's contiguous slice of the current maps is staged in shared memory by TMA bulk
//                     copies once per level; per iteration: batched model-map gathers, warp transpose-reduce, one 128-byte partial
//                     per CTA, ONE grid barrier, then every CTA sums the partials in the same fixed order and solves the 6x6
//                     system redundantly in FP64 (kt_solve.cuh) -- no second barrier, no pose broadcast, bit-identical poses;
//   icp_kernel        one launch per ITERATION (grid sized to the SM count, last-CTA tail solves): the operator API (kt_op_icp_step)
//                     and the fallback of the per-iteration RGB-D path.
// Reductions run in a fixed order (deterministic run to run); no host round trip inside a frame.
// Bound: latency of the per-iteration tail (barrier, partial sum, FP64 solve); the main phase is issue-bound; 48 B/pixel/iteration
// (24 streamed from the shared-memory stage + 24 gathered from L2), far from HBM-bound at 640x480.
#include "kt_ops.h"
#include "kt_solve.cuh"
#include "kt_reduce.cuh"
#include "kt_frame.cuh"

namespace kt {

namespace {

enum { ICP_THREADS = RED_THREADS };

struct IcpParams {
    IcpLevelArgs a;
    OdomState* st;
    float* partials;       // [gridDim.x][32]
    float* trace;          // [iter][44] or null
    int mode;              // 0 reduce only, 1 reduce + solve (ICP-only odometry)
};

__global__ void __launch_bounds__(ICP_THREADS)
icp_kernel(const IcpParams p)
{
    __shared__ float s_pose[24];
    __shared__ float s_red[ICP_THREADS / 32][32];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
    if (tid < 9) { s_pose[tid] = p.st->Rcurr[tid]; s_pose[12 + tid] = p.st->Rprev_inv[tid]; }
    if (tid < 3) { s_pose[9 + tid] = p.st->tcurr[tid]; s_pose[21 + tid] = p.st->tprev[tid]; }
    __syncthreads();
    const Mat33 Rcurr = mat33_rows(s_pose), Rprev_inv = mat33_rows(s_pose + 12);
    const float3 tcurr = make_float3(s_pose[9], s_pose[10], s_pose[11]), tprev = make_float3(s_pose[21], s_pose[22], s_pose[23]);

    const int cols = p.a.cols, rows = p.a.rows, N = cols * rows;
    const float* __restrict__ vmap_curr = p.a.vmap_curr;
    const float* __restrict__ nmap_curr = p.a.nmap_curr;
    const float* __restrict__ vmap_g_prev = p.a.vmap_g_prev;
    const float* __restrict__ nmap_g_prev = p.a.nmap_g_prev;
    const Intr intr = p.a.k;

    float sum[NSUM];
#pragma unroll
    for (int k = 0; k < NSUM; ++k) sum[k] = 0.f;

    for (int i = blockIdx.x * ICP_THREADS + tid; i < N; i += gridDim.x * ICP_THREADS) {
        const float3 vc = make_float3(__ldg(&vmap_curr[i]), __ldg(&vmap_curr[i + N]), __ldg(&vmap_curr[i + 2 * N]));
        const float3 nc = make_float3(__ldg(&nmap_curr[i]), __ldg(&nmap_curr[i + N]), __ldg(&nmap_curr[i + 2 * N]));
        icp_pixel(vc, nc, N, cols, rows, vmap_g_prev, nmap_g_prev, intr, Rcurr, tcurr, Rprev_inv, tprev, p.a.dist_thres, p.a.angle_thres, sum);
    }

    if (!grid_reduce29(sum, p.partials, &p.st->blocks_done, s_red, &s_last)) return;

    // ---- last CTA: the Gauss-Newton step ----
    if (tid < NSUM) p.st->sums_icp[tid] = s_red[0][tid];
    if (tid == 0) {
        OdomState* st = p.st;
        float A[36], b[6];
        unpack_normal_equations(s_red[0], A, b);
        if (p.trace) {
            float* t = p.trace + (size_t)st->iter * TRACE_STRIDE;
            for (int k = 0; k < 36; ++k) t[k] = A[k];
            for (int k = 0; k < 6; ++k) t[36 + k] = b[k];
            t[42] = s_red[0][27]; t[43] = s_red[0][28];
        }
        if (p.mode == 1) {
            double dA[36], db[6];
            for (int k = 0; k < 36; ++k) dA[k] = A[k];
            for (int k = 0; k < 6; ++k) db[k] = b[k];
            gauss_newton_update(dA, db, st);
            st->iter += 1;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Whole-frame ICP: all levels and iterations in ONE cooperative launch (one CTA per SM).  Per iteration:
//   main     every thread's pixels in batches of ICP_BATCH: project all, issue all model-map gathers, finish all (the projected point and
//            the current vertex stay in registers between the two halves); 29 sums per thread;
//   reduce   warp transpose-sum (lane l ends with component l) -> shared memory -> warp 0 adds the 16 warps in a fixed order;
//   exchange warp 0: ONE fire-and-forget 64-bit atomic per component into self-counting fixed-point words, poll until all CTAs are
//            in (grid_sum_words, kt_frame.cuh): no grid barrier, no fence, no re-read of 132 partials;
//   solve    lane 0 of warp 0 of EVERY CTA: the same FP64 LDL^T + Rodrigues + pose composition on the same bit-identical totals
//            (kt_solve.cuh, latency-trimmed form), so no pose broadcast is needed and all CTAs hold identical poses.
// Two __syncthreads per iteration.  The totals are exact integer sums => deterministic run to run.
// ICP_BATCH = pixels per thread whose model-map gathers are in flight together (template parameter: 4, or 5 when the level-0 share of a
// thread is 4 passes + a remainder -- 640x480 on 132 SMs: 4.55 pixels per thread -- so that the remainder does not cost a second batch's
// worth of L2 latency per iteration; the sums are accumulated in pass order either way, so the result does not depend on it)

struct IcpFrameParams {
    IcpLevelArgs lv[LEVELS];
    int iters[LEVELS];
    float pose12[12];          // Rprev (9), tprev (3)
    OdomState* st;
    unsigned long long* xwords;    // grid_sum_words exchange words (XW_WORDS), zero at launch
    float* trace;
    int* timeout;              // set to 1 if a peer CTA never arrived (bounded poll)
    long long* prof;           // optional: clock64() stamps per iteration from CTA 0 (debug)
    int stage_k;               // passes of FRAME_THREADS pixels per CTA held in the shared-memory stage (0 = no staging); a level with
                               // more passes stages its first stage_k and reads the rest from global memory
    float* host_pose; unsigned int host_seq;      // optional mapped host record: pose (12), time-out (1), sequence number (1)
    PeerWords pw; int rank;                       // pw.world > 1: the pixel rows are split over the ranks of a shared volume (grid_sum_words_mg)
};

template <int ICP_BATCH>
__global__ void __launch_bounds__(FRAME_THREADS, 1)
icp_frame_kernel(const IcpFrameParams p)
{
    extern __shared__ __align__(128) float s_stage[];               // [6 planes][stage_k][FRAME_THREADS]
    __shared__ FramePose s_pose;
    __shared__ float s_red[FRAME_THREADS / 32][32];
    __shared__ double s_sumd[32];
    __shared__ __align__(8) unsigned long long s_mbar;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int G = gridDim.x;
    Mat33 Rprev_inv; float3 tprev;
    frame_begin(s_pose, p.pose12, &s_mbar, Rprev_inv, tprev);

    GridSumState gs; gs.prev[0] = 0ull; gs.prev[1] = 0ull;
    int trace_a, trace_b;                    // where lane l's component lands in a trace record
    trace_slots(lane, trace_a, trace_b);
    int it = 0;
    unsigned int stage_parity = 0;
    for (int level = LEVELS - 1; level >= 0; --level) {
        if (p.iters[level] == 0) continue;
        const IcpLevelArgs& a = p.lv[level];
        const int cols = a.cols, rows = a.rows, N = cols * rows;
        const float* __restrict__ vmap_curr = a.vmap_curr;
        const float* __restrict__ nmap_curr = a.nmap_curr;
        const float* __restrict__ vmap_g_prev = a.vmap_g_prev;
        const float* __restrict__ nmap_g_prev = a.nmap_g_prev;
        const Intr intr = a.k;
        const float dist_thres = a.dist_thres, angle_thres = a.angle_thres;
        // pixels of this CTA: ONE contiguous range of q = ceil(N / G) pixels (rounded up to the 16-byte TMA granule), so that every SM
        // gets the same share
        // (split over the ranks of a shared volume: world * G CTAs, this one is number rank * G + blockIdx.x)
        const int GT = G * p.pw.world, gci = p.rank * G + (int)blockIdx.x;
        const int q = (((N + GT - 1) / GT) + 3) & ~3;
        const int i_begin = min(N, gci * q), cnt = min(N, i_begin + q) - i_begin;
        const int n_pass = (q + FRAME_THREADS - 1) / FRAME_THREADS;
        const int ps = p.stage_k * FRAME_THREADS;                    // floats per staged plane
        const bool staged = (p.stage_k > 0) && ((N & 3) == 0);
        const int n_st = staged ? min(n_pass, p.stage_k) : 0;       // passes read from shared memory; passes n_st.. come from global memory
        if (staged) {
            // The current vertex / normal maps do not change during the level's iterations: ONE bulk copy per plane (16-byte aligned)
            // brings the CTA's range -- its first n_st passes when the range is larger than the stage -- into shared memory through the
            // TMA engine; every iteration then reads its 24 streamed bytes per pixel from shared memory instead of L2.
            __syncthreads();                                         // previous level's readers are done with the stage
            if (tid == 0) {
                const unsigned int bytes = (unsigned int)min(cnt, n_st * FRAME_THREADS) * 4u;
                mbar_expect_tx(&s_mbar, bytes * 6u);                 // 0 completes the phase for CTAs without pixels at this level
                if (bytes) {
#pragma unroll
                    for (int pl = 0; pl < 3; ++pl) {
                        tma_bulk_g2s(&s_stage[pl * ps], vmap_curr + (size_t)pl * N + i_begin, bytes, &s_mbar);
                        tma_bulk_g2s(&s_stage[(3 + pl) * ps], nmap_curr + (size_t)pl * N + i_begin, bytes, &s_mbar);
                    }
                }
            }
            mbar_wait(&s_mbar, stage_parity);
            stage_parity ^= 1u;
        }
        for (int iter = 0; iter < p.iters[level]; ++iter, ++it) {
            const Mat33 Rcurr = mat33_rows(s_pose.R);
            const float3 tcurr = make_float3(s_pose.t[0], s_pose.t[1], s_pose.t[2]);
            const bool prof = (p.prof != 0) && blockIdx.x == 0 && tid == 0 && it < 64;
            if (prof) p.prof[it * 8 + 0] = clock64();
            float sum[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) sum[k] = 0.f;
            if (staged) {
                for (int k0 = 0; k0 < n_pass; k0 += ICP_BATCH) {
                    if (k0 * FRAME_THREADS + wid * 32 >= cnt) break;              // warp-uniform: this warp has no pixel in this batch
                    int j[ICP_BATCH]; float g[ICP_BATCH][6]; float3 vg[ICP_BATCH], vcp[ICP_BATCH];
#pragma unroll
                    for (int b = 0; b < ICP_BATCH; ++b) {
                        const int o = (k0 + b) * FRAME_THREADS + tid;
                        j[b] = -1;
                        if (k0 + b < n_pass && o < cnt) {
                            const float3 vc = k0 + b < n_st ? make_float3(s_stage[o], s_stage[ps + o], s_stage[2 * ps + o])
                                                            : make_float3(__ldg(&vmap_curr[i_begin + o]), __ldg(&vmap_curr[i_begin + o + N]), __ldg(&vmap_curr[i_begin + o + 2 * N]));
                            j[b] = icp_pixel_project(vc, cols, rows, intr, Rcurr, tcurr, Rprev_inv, tprev, vg[b], vcp[b]);
                        }
                    }
#pragma unroll
                    for (int b = 0; b < ICP_BATCH; ++b) {
                        const int jj = j[b] < 0 ? 0 : j[b];
                        g[b][0] = __ldg(&vmap_g_prev[jj]); g[b][1] = __ldg(&vmap_g_prev[jj + N]); g[b][2] = __ldg(&vmap_g_prev[jj + 2 * N]);
                        g[b][3] = __ldg(&nmap_g_prev[jj]); g[b][4] = __ldg(&nmap_g_prev[jj + N]); g[b][5] = __ldg(&nmap_g_prev[jj + 2 * N]);
                    }
#pragma unroll
                    for (int b = 0; b < ICP_BATCH; ++b) {
                        if (j[b] >= 0) {
                            const int o = (k0 + b) * FRAME_THREADS + tid;
                            const float3 nc = k0 + b < n_st ? make_float3(s_stage[3 * ps + o], s_stage[4 * ps + o], s_stage[5 * ps + o])
                                                            : make_float3(__ldg(&nmap_curr[i_begin + o]), __ldg(&nmap_curr[i_begin + o + N]), __ldg(&nmap_curr[i_begin + o + 2 * N]));
                            icp_pixel_finish(vg[b], vcp[b], nc,
                                              make_float3(g[b][0], g[b][1], g[b][2]), make_float3(g[b][3], g[b][4], g[b][5]),
                                              Rcurr, Rprev_inv, tprev, dist_thres, angle_thres, sum);
                        }
                    }
                }
            } else {
                for (int i = gci * FRAME_THREADS + tid; i < N; i += GT * FRAME_THREADS) {
                    const float3 vc = make_float3(__ldg(&vmap_curr[i]), __ldg(&vmap_curr[i + N]), __ldg(&vmap_curr[i + 2 * N]));
                    const float3 nc = make_float3(__ldg(&nmap_curr[i]), __ldg(&nmap_curr[i + N]), __ldg(&nmap_curr[i + 2 * N]));
                    icp_pixel(vc, nc, N, cols, rows, vmap_g_prev, nmap_g_prev, intr, Rcurr, tcurr, Rprev_inv, tprev, dist_thres, angle_thres, sum);
                }
            }
            // CTA reduction: warp transpose-sum (lane l ends with component l), then warp 0 adds the 16 warps in a fixed order
            {
                const float v = warp_transpose_sum(sum, lane);
                s_red[wid][lane] = v;
            }
            __syncthreads();
            if (wid == 0) {
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < FRAME_THREADS / 32; ++w) v += s_red[w][lane];
                if (prof) p.prof[it * 8 + 1] = clock64();
                const double total = p.pw.world > 1 ? grid_sum_words_mg(p.pw, p.rank, it, lane, v, gs, (unsigned int)GT, p.timeout)
                                                    : grid_sum_words(p.xwords, it, lane, v, gs, (unsigned int)G, p.timeout);
                s_sumd[lane] = total;
                __syncwarp();
                if (prof) p.prof[it * 8 + 2] = clock64();
                if (lane == 0) {
                    double dA[36], db[6];
                    unpack_normal_equations(s_sumd, dA, db);
                    gauss_newton_update_fast(dA, db, s_pose.Rt, s_pose.Rp, s_pose.tp, s_pose.R, s_pose.t);
                    if (prof) p.prof[it * 8 + 3] = clock64();
                }
                if (p.trace && blockIdx.x == 0 && it < 64) {
                    // the iteration's normal equations as the reference hands them to the host (reduce.cu:404-418); CTA 0 is on the critical
                    // path of every exchange, so the component -> slot mapping was worked out once per launch (trace_a / trace_b)
                    float* t = p.trace + (size_t)it * TRACE_STRIDE;
                    const float value = (float)total;
                    if (trace_a >= 0) t[trace_a] = value;
                    if (trace_b >= 0) t[trace_b] = value;
                }
            }
            __syncthreads();
        }
    }
    frame_end(s_pose, it, p.st, p.host_pose, p.host_seq, p.timeout);
}

__global__ void odom_begin_kernel(OdomState* st, const float* pose12)
{
    // pose12: Rprev (9) tprev (3), uploaded by the host (it owns rmats_/tvecs_ like the reference tracker)
    if (threadIdx.x == 0) {
        for (int k = 0; k < 9; ++k) { st->Rprev[k] = pose12[k]; st->Rcurr[k] = pose12[k]; }
        for (int k = 0; k < 3; ++k) { st->tprev[k] = pose12[9 + k]; st->tcurr[k] = pose12[9 + k]; }
        mat3f_inverse(st->Rprev, st->Rprev_inv);                       // Rprev.inverse(), ICPOdometry.cpp:81
        for (int k = 0; k < 16; ++k) st->resultRt[k] = (k % 5 == 0) ? 1.0 : 0.0;
        st->iter = 0; st->blocks_done = 0; st->blocks_done_rgb = 0;
        st->rgb_count = 0; st->rgb_sigma = 0;
    }
}

} // namespace

static int sm_count() { return device_info().sm_count; }

int reduce_grid_for(int n_items)
{
    // two items per thread are enough to cover latency; cap at 4 CTAs per SM (a multiple of the SM count) and MAX_PARTIALS
    int want = div_up(n_items, RED_THREADS * 2);
    int cap = sm_count() * 4;
    if (cap > MAX_PARTIALS) cap = MAX_PARTIALS;
    return want < cap ? (want < 1 ? 1 : want) : cap;
}

int icp_iteration(const IcpLevelArgs& a, OdomState* state, float* partials, float* trace, int mode, cudaStream_t s)
{
    IcpParams p; p.a = a; p.st = state; p.partials = partials; p.trace = trace; p.mode = mode;
    int grid = reduce_grid_for(a.rows * a.cols);
    icp_kernel<<<grid, ICP_THREADS, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

int odom_begin_frame(OdomState* state, const float* pose12_dev, cudaStream_t s)
{
    odom_begin_kernel<<<1, 32, 0, s>>>(state, pose12_dev);
    KT_LAUNCH_CHECK();
    return 0;
}


// Whole-frame ICP (ICP-only odometry).  pose12 = Rprev (9) + tprev (3) on the host; the result lands in state->Rcurr/tcurr.
// xwords_dev: XW_WORDS 64-bit exchange words, ZERO when the launch starts (the tracker resets them once per frame, kt_tracker.cu).
int icp_frame(const IcpLevelArgs* levels, const int* iters, const float* pose12_host, OdomState* state, unsigned long long* xwords_dev,
              float* trace, int* timeout_dev, long long* prof_dev, float* host_pose, unsigned int host_seq, cudaStream_t s,
              unsigned long long* const* peer_words, int world, int rank)
{
    IcpFrameParams p;
    p.pw.world = (peer_words && world > 1) ? world : 1; p.rank = p.pw.world > 1 ? rank : 0;
    for (int g = 0; g < 8; ++g) p.pw.w[g] = (p.pw.world > 1 && g < world) ? peer_words[g] : xwords_dev;
    p.host_pose = host_pose; p.host_seq = host_seq;
    p.prof = prof_dev;
    for (int l = 0; l < LEVELS; ++l) { p.lv[l] = levels[l]; p.iters[l] = iters[l]; }
    for (int k = 0; k < 12; ++k) p.pose12[k] = pose12_host[k];
    p.st = state; p.xwords = xwords_dev; p.trace = trace; p.timeout = timeout_dev;
    const int grid = frame_grid();
    // shared-memory stage for the current maps: 6 planes x stage_k x 2 KB (one contiguous pixel range per CTA), sized for the largest level in use
    int need_k = 0;
    for (int l = 0; l < LEVELS; ++l)
        if (iters[l] > 0) { int q = (div_up(levels[l].rows * levels[l].cols, grid * p.pw.world) + 3) & ~3; int k = div_up(q, FRAME_THREADS); if (k > need_k) need_k = k; }
    DeviceInfo& di = device_info();
    const int smem_optin = di.smem_optin;
    if (!(di.configured & 1u)) {
        if (smem_optin > 0) {
            cudaFuncSetAttribute((const void*)icp_frame_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin - 4096);
            cudaFuncSetAttribute((const void*)icp_frame_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin - 4096);
        }
        di.configured |= 1u;
    }
    // the stage holds as many passes as the largest level needs, up to what a block's shared memory takes (STAGE_MAX_K on an H100);
    // a level that needs more stages that many and streams the rest (1280x960 level 0 on 132 SMs: 18 of 19 passes)
    int stage_k = need_k < STAGE_MAX_K ? need_k : STAGE_MAX_K;
    const int smem_k = smem_optin > 4096 ? (smem_optin - 4096) / (6 * FRAME_THREADS * (int)sizeof(float)) : 0;
    if (stage_k > smem_k) stage_k = smem_k;
    static int stage_knob = -1;                     // KT_ICP_STAGE_PASSES (test hook): a smaller stage, so that 640x480 takes the partial path
    if (stage_knob < 0) { const char* e = getenv("KT_ICP_STAGE_PASSES"); stage_knob = e ? atoi(e) : 0; }
    if (stage_knob > 0 && stage_k > stage_knob) stage_k = stage_knob;
    if (stage_k < 0) stage_k = 0;
    const size_t stage_bytes = (size_t)6 * stage_k * FRAME_THREADS * sizeof(float);
    const bool can_stage = stage_k > 0;
    p.stage_k = stage_k;
    const int batch = (need_k % 4 == 1) ? 5 : 4;    // 5 when the largest level leaves a remainder pass after groups of 4
    void* args[] = {&p};
    const void* fn = batch == 5 ? (const void*)icp_frame_kernel<5> : (const void*)icp_frame_kernel<4>;
    cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(FRAME_THREADS), args, can_stage ? stage_bytes : 0, s);
    ++g_launches;
    if (e != cudaSuccess) return cuda_check(e, "cudaLaunchCooperativeKernel(icp_frame_kernel)", __FILE__, __LINE__);
    return 0;
}

namespace { __global__ void __launch_bounds__(64) zero_words_kernel(unsigned long long* w, int n, int stride) { for (int i = threadIdx.x; i < n; i += blockDim.x) w[(size_t)i * stride] = 0ull; } }

size_t odom_exchange_words() { return (size_t)XW_WORDS; }
int odom_exchange_used(int* stride) { if (stride) *stride = XW_STRIDE; return XW_SETS * 32; }

int odom_exchange_reset(unsigned long long* xwords_dev, cudaStream_t s)
{
    zero_words_kernel<<<1, 64, 0, s>>>(xwords_dev, XW_SETS * 32, XW_STRIDE);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
