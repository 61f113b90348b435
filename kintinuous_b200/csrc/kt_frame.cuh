// kintinuous_b200 -- device helpers shared by the whole-frame (persistent, cooperative) odometry kernels:
// grid-wide exchange, TMA bulk-copy staging, warp transpose-reduce, launch set-up and hand-over, and the point-to-plane ICP pixel that
// the per-iteration icp_kernel evaluates too.
#pragma once
#include "kt_ops.h"
#include "kt_reduce.cuh"
#include "kt_solve.cuh"

namespace kt {

enum { FRAME_THREADS = 512, STAGE_MAX_K = 18 };   // 18 passes x 6 planes x 2 KB = 216 KB: the most an H100 block's 227 KB take beside the static smem

// ---- grid-wide sum of the CTAs' 29 partial sums without a barrier, a fence or a second pass over per-CTA partials ----
// One 64-bit word per component (two sets, by iteration parity; XW_STRIDE 8-byte units apart so that the words live in different L2
// slices: 2400 cycles per exchange at 1280 B against 3700 with the words packed).  Every CTA adds  round(partial * 2^32) with the low 8 bits cleared, plus 1  to the word with ONE fire-and-forget atomic: the
// low byte of (word now - word when this set was last complete) therefore counts the CTAs that have arrived, and the rest is the exact
// integer sum of their partials.  Integer addition commutes, so the total is bit-identical in every CTA and from run to run whatever
// the arrival order; its resolution (2^-24 absolute per CTA) is finer than the float partials' own rounding for every entry that
// matters to the solve (DESIGN.md section 3.2).  Latency: one atomic to L2 plus one poll round trip after the LAST CTA arrived
// (measured with tools/tail_bench.cu against the counter barrier + partial re-read it replaces).
// Requirements: gridDim.x <= 255 (frame_grid); the words are zero when the launch starts (the host keeps them so, kt_tracker.cu).
// Range: a signed 64-bit word holds round(x * 2^32), so the exchange is exact only while every per-CTA partial and every grid total stays
// below 2^31 in magnitude; past that __double2ll_rn saturates, the word wraps, and the count byte still completes, so nothing would flag
// it.  The ICP sums (icp_frame_kernel, exchange 1 of rgbd_frame_kernel) stay below that by geometry: every row entry is bounded by the
// camera-to-surface distance, at most the volume's diagonal, so the largest sum is about N * 3 * volume_size^2 -- 1.3e8 for a 6 m volume
// at 1280x960, 16x below the limit (a volume above ~25 m could reach it).  The photometric sums have no such bound (with sigma = 1, as
// on a repeated frame, a 640x480 level-0 entry reaches ~8e12): exchange 2 of rgbd_frame_kernel carries them through grid_sum_words_wide.
// Word sets: an exchange with counter ex uses set (ex & 1) -- the words of grid_sum_fixed, or the high words of grid_sum_words_wide --
// and a wide exchange also set 2 + (ex & 1) for its low words.  icp_frame_kernel exchanges once per iteration (sets 0 and 1).
// rgbd_frame_kernel exchanges twice per iteration from ex = 0, so exchange 1 (one word) always lands on set 0 and the wide exchange 2 on
// sets 1 and 3; set 2 stays unused there.  It is kept so that grid_sum_words_wide, like grid_sum_fixed, is correct on consecutive
// exchanges (tools/tail_bench.cu runs it so), not only when another exchange separates two wide ones.
enum { XW_STRIDE = 160, XW_SETS = 4, XW_WORDS = XW_SETS * 32 * XW_STRIDE };     // 1280 B apart (tools/tail_bench.cu times other strides)

__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v)
{ asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p)
{ unsigned long long v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }

struct GridSumState { unsigned long long prev[2]; };          // per lane: the word's value when its set was last complete

// Called by ALL 32 lanes of ONE warp per CTA.  Lanes with active == true contribute q (an integer whose low 8 bits are zero) to their
// word and get the grid total of their word back; `ex` = exchange counter of the launch (its parity selects the word set; a CTA can be
// at most one exchange ahead of another, so two sets suffice).  A lost peer would spin forever: the poll is bounded (~2 s at 2 GHz) and
// reports through *timeout instead of hanging the GPU.
__device__ __forceinline__ long long grid_sum_fixed(unsigned long long* words, int ex, int lane, bool active, long long q, GridSumState& st, unsigned int G, int* timeout)
{
    long long total = 0;
    if (active) {
        const int par = ex & 1;
        unsigned long long* w = words + ((size_t)par * 32 + lane) * XW_STRIDE;
        red_add_u64(w, (unsigned long long)(q + 1));
        const unsigned long long prev = par ? st.prev[1] : st.prev[0];
        unsigned long long now, d;
        unsigned int spins = 0; long long t0 = 0;
        for (;;) {
            now = ld_relaxed_u64(w); d = now - prev;
            if ((unsigned int)(d & 0xFFull) == G) break;
            if ((++spins & 0x3FFFu) == 0) {
                const long long t = clock64();
                if (t0 == 0) t0 = t;
                else if (t - t0 > 4000000000LL) { if (timeout) *timeout = 1; break; }
            }
        }
        if (par) st.prev[1] = now; else st.prev[0] = now;
        total = (long long)(d - (unsigned long long)G);
    }
    return total;
}
__device__ __forceinline__ long long to_fixed32(float v) { return __double2ll_rn((double)v * 4294967296.0) & ~0xFFll; }
__device__ __forceinline__ double from_fixed32(long long t) { return (double)t * (1.0 / 4294967296.0); }

// The usual case: lane l < 29 passes the CTA's partial of component l and gets the grid total of component l back (as a double: the
// exact integer sum scaled by 2^-32).
__device__ __forceinline__ double grid_sum_words(unsigned long long* words, int ex, int lane, float partial, GridSumState& st, unsigned int G, int* timeout)
{
    return from_fixed32(grid_sum_fixed(words, ex, lane, lane < NSUM, to_fixed32(partial), st, G, timeout));
}

// grid_sum_words over two self-counting words per component, for partials beyond the 2^31 range of one: hi = rint(partial) in units of 1
// (shifted past the count byte) and lo = to_fixed32(partial - hi), where partial - hi is exact in float.  hi * 2^32 + lo equals
// to_fixed32(partial) exactly whenever that is in range, and the total hi_tot + lo_tot * 2^-32 is ONE correctly rounded double addition of
// the same exact integer sum scaled by 2^-32, so every result grid_sum_words could represent comes back bit-identical; the range grows to
// 2^55.  st_lo keeps the low words' state as st keeps the high words'.  Both words are added, then polled together: one round trip.
__device__ __forceinline__ double grid_sum_words_wide(unsigned long long* words, int ex, int lane, float partial, GridSumState& st, GridSumState& st_lo,
                                                      unsigned int G, int* timeout)
{
    if (lane >= NSUM) return 0.0;
    const int par = ex & 1;
    unsigned long long* wh = words + ((size_t)par * 32 + lane) * XW_STRIDE;
    unsigned long long* wl = words + ((size_t)(2 + par) * 32 + lane) * XW_STRIDE;
    const float hi = rintf(partial);
    red_add_u64(wh, (unsigned long long)(__float2ll_rn(hi) * 256 + 1));
    red_add_u64(wl, (unsigned long long)(to_fixed32(partial - hi) + 1));
    const unsigned long long prev_h = par ? st.prev[1] : st.prev[0], prev_l = par ? st_lo.prev[1] : st_lo.prev[0];
    unsigned long long now_h, now_l, dh, dl;
    unsigned int spins = 0; long long t0 = 0;
    for (;;) {
        now_h = ld_relaxed_u64(wh); now_l = ld_relaxed_u64(wl);
        dh = now_h - prev_h; dl = now_l - prev_l;
        if ((unsigned int)(dh & 0xFFull) == G && (unsigned int)(dl & 0xFFull) == G) break;
        if ((++spins & 0x3FFFu) == 0) {
            const long long t = clock64();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 4000000000LL) { if (timeout) *timeout = 1; break; }
        }
    }
    if (par) { st.prev[1] = now_h; st_lo.prev[1] = now_l; } else { st.prev[0] = now_h; st_lo.prev[0] = now_l; }
    return (double)((long long)(dh - (unsigned long long)G) >> 8) + from_fixed32((long long)(dl - (unsigned long long)G));
}


// ---- the same exchange ACROSS GPUs (shared-volume mode with the pixel rows of every level split over the ranks): every CTA of every rank
// adds its partial to the word of EVERY rank -- one system-scope red.add per rank over NVLink peer memory, fire-and-forget -- and polls its
// LOCAL word until all world * G contributions are in.  This is the north_star's per-iteration all-reduce of the 29 normal-equation sums,
// fused into the kernel: no collective library call, no second kernel, and because integer addition commutes every rank reads
// bit-identical totals (hence identical poses) whatever the arrival order.  12 count bits (up to 4095 CTAs), so partials are rounded to
// 2^-20 instead of 2^-24 (still far below the float partials' own rounding for every entry that matters to the solve).
__device__ __forceinline__ void red_add_sys_u64(unsigned long long* p, unsigned long long v)
{ asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p)
{ unsigned long long v; asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }

struct PeerWords { unsigned long long* w[8]; int world; };

__device__ __forceinline__ double grid_sum_words_mg(const PeerWords& pw, int rank, int ex, int lane, float partial, GridSumState& st, unsigned int G_total, int* timeout)
{
    long long total = 0;
    if (lane < NSUM) {
        const int par = ex & 1;
        const size_t off = ((size_t)par * 32 + lane) * XW_STRIDE;
        const long long q = __double2ll_rn((double)partial * 4294967296.0) & ~0xFFFll;
        for (int g = 0; g < pw.world; ++g) red_add_sys_u64(pw.w[g] + off, (unsigned long long)(q + 1));
        const unsigned long long* w = pw.w[rank] + off;
        const unsigned long long prev = par ? st.prev[1] : st.prev[0];
        unsigned long long now, d;
        unsigned int spins = 0; long long t0 = 0;
        for (;;) {
            now = ld_relaxed_sys_u64(w); d = now - prev;
            if ((unsigned int)(d & 0xFFFull) == G_total) break;
            if ((++spins & 0x3FFFu) == 0) {
                const long long t = clock64();
                if (t0 == 0) t0 = t;
                else if (t - t0 > 4000000000LL) { if (timeout) *timeout = 1; break; }
            }
        }
        if (par) st.prev[1] = now; else st.prev[0] = now;
        total = (long long)(d - (unsigned long long)G_total);
    }
    return from_fixed32(total);
}

// ---- TMA (bulk async copy engine) helpers: global -> shared 1-D bulk copies completing on an mbarrier ----
__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned int bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, unsigned int bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned int parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "KT_WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra KT_WAIT_DONE;\n"
        "bra KT_WAIT_LOOP;\n"
        "KT_WAIT_DONE:\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}

// 32 per-lane values -> lane l holds the warp total of value l (31 shuffles instead of 32 x 5; fixed tree).  One template instance per
// step, so that every index into v is a compile-time constant: with the step as a loop variable nvcc leaves the loop rolled in the
// whole-frame kernels, which puts v -- the thread's running sums, updated for every pixel -- in local memory (DESIGN.md section 3.2).
template <int STEP>
__device__ __forceinline__ void warp_transpose_step(float (&v)[32], int lane)
{
    const bool upper = (lane & STEP) != 0;
#pragma unroll
    for (int j = 0; j < STEP; ++j) {
        const float send = upper ? v[j] : v[j + STEP];
        const float keep = upper ? v[j + STEP] : v[j];
        v[j] = keep + __shfl_xor_sync(0xffffffffu, send, STEP);
    }
}
__device__ __forceinline__ float warp_transpose_sum(float (&v)[32], int lane)
{
    warp_transpose_step<16>(v, lane);
    warp_transpose_step<8>(v, lane);
    warp_transpose_step<4>(v, lane);
    warp_transpose_step<2>(v, lane);
    warp_transpose_step<1>(v, lane);
    return v[0];
}

// ---- the point-to-plane ICP pixel (ICPReduction::search + getProducts, cuda/reduce.cu:211-316) ----
// Split in two so that the model-map gathers of several pixels can be in flight together (the per-iteration time of the whole-frame
// kernel is the latency of these dependent L2 loads, not their bandwidth):
//   icp_pixel_project  current vertex -> index of the model pixel it projects to, or -1      (reduce.cu:222-240); hands over vcurr_g
//                      (volume frame) and vcurr_cp (previous camera frame; it IS s_cp of reduce.cu:268 -- the same expression)
//   icp_pixel_finish   tests + row products from the six gathered floats                     (reduce.cu:241-316)
// Q16: a NaN current vertex is rejected before the model map is read; the reference rejects it through NaN propagation.
__device__ __forceinline__ int icp_pixel_project(const float3& vcurr, int cols, int rows, const Intr& intr,
                                                 const Mat33& Rcurr, const float3& tcurr, const Mat33& Rprev_inv, const float3& tprev,
                                                 float3& vcurr_g, float3& vcurr_cp)
{
    if (isnan(vcurr.x)) return -1;
    vcurr_g = add3(mul33(Rcurr, vcurr), tcurr);
    vcurr_cp = mul33(Rprev_inv, sub3(vcurr_g, tprev));
    int2 ukr;
    ukr.x = __float2int_rn(vcurr_cp.x * intr.fx / vcurr_cp.z + intr.cx);
    ukr.y = __float2int_rn(vcurr_cp.y * intr.fy / vcurr_cp.z + intr.cy);
    if (ukr.x < 0 || ukr.y < 0 || ukr.x >= cols || ukr.y >= rows || vcurr_cp.z < 0) return -1;
    return ukr.y * cols + ukr.x;
}

template <int S>
__device__ __forceinline__ void icp_pixel_finish(const float3& vcurr_g, const float3& s_cp, const float3& ncurr, const float3& vprev_g, const float3& nprev_g,
                                                 const Mat33& Rcurr, const Mat33& Rprev_inv, const float3& tprev,
                                                 float dist_thres, float angle_thres, float (&sum)[S])
{
    if (isnan(vprev_g.x) || isnan(nprev_g.x) || isnan(ncurr.x)) return;
    float3 ncurr_g = mul33(Rcurr, ncurr);
    float dist = norm3(sub3(vprev_g, vcurr_g));
    float sine = norm3(cross3(ncurr_g, nprev_g));
    if (!(sine < angle_thres && dist <= dist_thres)) return;
    float3 d_cp = mul33(Rprev_inv, sub3(vprev_g, tprev));
    float3 n_cp = mul33(Rprev_inv, nprev_g);
    float3 sxn = cross3(s_cp, n_cp);
    const float row[7] = {n_cp.x, n_cp.y, n_cp.z, sxn.x, sxn.y, sxn.z, dot3(n_cp, sub3(s_cp, d_cp))};
    accumulate_row(sum, row);
}

// One pixel at a time: project, gather the model pixel (planes N floats apart), finish.
template <int S>
__device__ __forceinline__ void icp_pixel(const float3& vcurr, const float3& ncurr, int N, int cols, int rows,
                                          const float* __restrict__ vmap_g_prev, const float* __restrict__ nmap_g_prev,
                                          const Intr& intr, const Mat33& Rcurr, const float3& tcurr, const Mat33& Rprev_inv, const float3& tprev,
                                          float dist_thres, float angle_thres, float (&sum)[S])
{
    // initialised although project sets them on every path that reaches finish: left undefined, they cost rgbd_frame_kernel<true>, at
    // its 128-register cap, 36 bytes of spills
    float3 vcurr_g = make_float3(0.f, 0.f, 0.f), vcurr_cp = vcurr_g;
    const int j = icp_pixel_project(vcurr, cols, rows, intr, Rcurr, tcurr, Rprev_inv, tprev, vcurr_g, vcurr_cp);
    if (j < 0) return;
    const float3 vprev_g = make_float3(__ldg(&vmap_g_prev[j]), __ldg(&vmap_g_prev[j + N]), __ldg(&vmap_g_prev[j + 2 * N]));
    const float3 nprev_g = make_float3(__ldg(&nmap_g_prev[j]), __ldg(&nmap_g_prev[j + N]), __ldg(&nmap_g_prev[j + 2 * N]));
    icp_pixel_finish(vcurr_g, vcurr_cp, ncurr, vprev_g, nprev_g, Rcurr, Rprev_inv, tprev, dist_thres, angle_thres, sum);
}

// ---- launch set-up and hand-over shared by icp_frame_kernel and rgbd_frame_kernel ----
// The pose every CTA keeps in shared memory; the redundant solves keep the copies of all CTAs bit-identical.
struct FramePose {
    float Rp[9], tp[3], Rpi[9];    // previous pose and Rprev.inverse()
    float R[9], t[3];              // running estimate
    double Rt[16];                 // resultRt (ICPOdometry.cpp:83)
};

__device__ __forceinline__ Mat33 mat33_rows(const float* m)
{
    Mat33 r; r.r0 = make_float3(m[0], m[1], m[2]); r.r1 = make_float3(m[3], m[4], m[5]); r.r2 = make_float3(m[6], m[7], m[8]); return r;
}

// pose12 = Rprev (9), tprev (3).  Thread 0 sets the pose, Rprev.inverse() (ICPOdometry.cpp:81), resultRt = I and the stage's mbarrier;
// then every thread takes Rprev^-1 and tprev into registers.
__device__ __forceinline__ void frame_begin(FramePose& fp, const float* pose12, unsigned long long* mbar, Mat33& Rprev_inv, float3& tprev)
{
    if (threadIdx.x == 0) {
        for (int k = 0; k < 9; ++k) { fp.Rp[k] = pose12[k]; fp.R[k] = pose12[k]; }
        for (int k = 0; k < 3; ++k) { fp.tp[k] = pose12[9 + k]; fp.t[k] = pose12[9 + k]; }
        mat3f_inverse(fp.Rp, fp.Rpi);
        for (int k = 0; k < 16; ++k) fp.Rt[k] = (k % 5 == 0) ? 1.0 : 0.0;
        mbar_init(mbar, 1);
    }
    __syncthreads();
    Rprev_inv = mat33_rows(fp.Rpi);
    tprev = make_float3(fp.tp[0], fp.tp[1], fp.tp[2]);
}

// CTA 0 writes the estimate and the iteration count to the OdomState.  With host_pose, the estimate also goes straight to mapped, pinned
// HOST memory (12 floats, the time-out flag, then a sequence number behind a system-scope fence): the host polls the sequence number
// instead of paying a D2H copy + stream synchronisation per frame.
__device__ __forceinline__ void frame_end(const FramePose& fp, int it, OdomState* st, float* host_pose, unsigned int host_seq, const int* timeout)
{
    const int tid = threadIdx.x;
    if (blockIdx.x != 0 || tid >= 12) return;
    if (tid < 9) st->Rcurr[tid] = fp.R[tid]; else st->tcurr[tid - 9] = fp.t[tid - 9];
    if (tid == 0) st->iter = it;
    if (host_pose && tid == 0) {
        volatile float* hp = host_pose;
        for (int k = 0; k < 9; ++k) hp[k] = fp.R[k];
        for (int k = 0; k < 3; ++k) hp[9 + k] = fp.t[k];
        ((volatile int*)host_pose)[12] = timeout ? *(volatile const int*)timeout : 0;
        __threadfence_system();
        ((volatile unsigned int*)host_pose)[13] = host_seq;
    }
}

// Where component c of the 29 sums lands in a trace record, A (6x6 row-major, symmetric) | b (6) | residual | inliers, as the reference
// hands the normal equations to the host (reduce.cu:404-418): the 27 products are the upper triangle with the b column, rows of 7, 6, 5, ...
// entries (internal.h:101-106).  An entry of A has two slots (a, b), every other component one (b = -1); c >= 29 has none.
__device__ __forceinline__ void trace_slots(int c, int& a, int& b)
{
    a = -1; b = -1;
    if (c >= NSUM) return;
    if (c >= 27) { a = 42 + (c - 27); return; }
    int i = 0, base = 0;
    while (c >= base + (7 - i) && i < 6) { base += 7 - i; ++i; }
    const int j = i + (c - base);
    if (j == 6) a = 36 + i; else { a = j * 6 + i; b = i * 6 + j; }
}

// Grid of a whole-frame kernel: one CTA per SM, at most 255 because the exchange words count arrivals in 8 bits (grid_sum_fixed).
inline int frame_grid()
{
    const int sms = device_info().sm_count;
    return sms < 255 ? sms : 255;
}

} // namespace kt
