// kintinuous_b200 -- device helpers shared by the whole-frame (persistent, cooperative) odometry kernels:
// grid barrier, TMA bulk-copy staging, warp transpose-reduce, the per-pixel point-to-plane row.
#pragma once
#include "kt_ops.h"
#include "kt_reduce.cuh"

namespace kt {

enum { FRAME_THREADS = 512, STAGE_MAX_K = 18 };   // 18 passes x 6 planes x 2 KB = 216 KB: the most an H100 block's 227 KB take beside the static smem

__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int target)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(bar, 1u);
        while ((int)(*((volatile unsigned int*)bar) - target) < 0) { }
        __threadfence();
    }
    __syncthreads();
}

// ---- grid-wide sum of the CTAs' 29 partial sums without a barrier, a fence or a second pass over per-CTA partials ----
// One 64-bit word per component (two sets, by iteration parity; XW_STRIDE 8-byte units apart so that the words live in different L2
// slices: 2400 cycles per exchange at 1280 B against 3700 with the words packed).  Every CTA adds  round(partial * 2^32) with the low 8 bits cleared, plus 1  to the word with ONE fire-and-forget atomic: the
// low byte of (word now - word when this set was last complete) therefore counts the CTAs that have arrived, and the rest is the exact
// integer sum of their partials.  Integer addition commutes, so the total is bit-identical in every CTA and from run to run whatever
// the arrival order; its resolution (2^-24 absolute per CTA) is finer than the float partials' own rounding for every entry that
// matters to the solve (DESIGN.md section 3.2).  Latency: one atomic to L2 plus one poll round trip after the LAST CTA arrived
// (measured with tools/tail_bench.cu against the counter barrier + partial re-read it replaces).
// Requirements: gridDim.x <= 255; the words are zero when the launch starts (the host keeps them so, kt_tracker.cu).
enum { XW_STRIDE = 160, XW_WORDS = 2 * 32 * XW_STRIDE };     // 1280 B apart (tools/tail_bench.cu times other strides)

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

// 32 per-lane values -> lane l holds the warp total of value l (31 shuffles instead of 32 x 5; fixed tree)
__device__ __forceinline__ float warp_transpose_sum(float (&v)[32], int lane)
{
#pragma unroll
    for (int step = 16; step >= 1; step >>= 1) {
        const bool upper = (lane & step) != 0;
#pragma unroll
        for (int j = 0; j < step; ++j) {
            const float send = upper ? v[j] : v[j + step];
            const float keep = upper ? v[j + step] : v[j];
            v[j] = keep + __shfl_xor_sync(0xffffffffu, send, step);
        }
    }
    return v[0];
}

// one pixel whose current vertex / normal were staged in shared memory
__device__ __forceinline__ void icp_pixel_staged(const float3& vcurr, const float3& ncurr, int N, int cols, int rows,
                                                 const float* __restrict__ vmap_g_prev, const float* __restrict__ nmap_g_prev,
                                                 const Intr& intr, const Mat33& Rcurr, const float3& tcurr, const Mat33& Rprev_inv, const float3& tprev,
                                                 float dist_thres, float angle_thres, float (&sum)[32])
{
    if (isnan(vcurr.x)) return;
    float3 vcurr_g = add3(mul33(Rcurr, vcurr), tcurr);
    float3 vcurr_cp = mul33(Rprev_inv, sub3(vcurr_g, tprev));
    int2 ukr;
    ukr.x = __float2int_rn(vcurr_cp.x * intr.fx / vcurr_cp.z + intr.cx);
    ukr.y = __float2int_rn(vcurr_cp.y * intr.fy / vcurr_cp.z + intr.cy);
    if (ukr.x < 0 || ukr.y < 0 || ukr.x >= cols || ukr.y >= rows || vcurr_cp.z < 0) return;
    const int j = ukr.y * cols + ukr.x;
    float3 vprev_g, nprev_g;
    vprev_g.x = __ldg(&vmap_g_prev[j]); vprev_g.y = __ldg(&vmap_g_prev[j + N]); vprev_g.z = __ldg(&vmap_g_prev[j + 2 * N]);
    nprev_g.x = __ldg(&nmap_g_prev[j]); nprev_g.y = __ldg(&nmap_g_prev[j + N]); nprev_g.z = __ldg(&nmap_g_prev[j + 2 * N]);
    if (isnan(vprev_g.x) || isnan(nprev_g.x) || isnan(ncurr.x)) return;
    float3 ncurr_g = mul33(Rcurr, ncurr);
    float dist = norm3(sub3(vprev_g, vcurr_g));
    float sine = norm3(cross3(ncurr_g, nprev_g));
    if (!(sine < angle_thres && dist <= dist_thres)) return;
    float3 s_cp = mul33(Rprev_inv, sub3(vcurr_g, tprev));
    float3 d_cp = mul33(Rprev_inv, sub3(vprev_g, tprev));
    float3 n_cp = mul33(Rprev_inv, nprev_g);
    float3 sxn = cross3(s_cp, n_cp);
    const float row[7] = {n_cp.x, n_cp.y, n_cp.z, sxn.x, sxn.y, sxn.z, dot3(n_cp, sub3(s_cp, d_cp))};
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 7; ++b) sum[k++] += row[a] * row[b];
    sum[27] += row[6] * row[6];
    sum[28] += 1.f;
}

// The same pixel split in two so that the model-map gathers of several pixels can be in flight together (the per-iteration time of
// the whole-frame kernel is the latency of these dependent L2 loads, not their bandwidth):
//   icp_pixel_project  current vertex -> index of the model pixel it projects to, or -1      (reduce.cu:222-240)
//   icp_pixel_finish   tests + row products from the six gathered floats                     (reduce.cu:241-316)
// Expression order is the one of icp_pixel_staged, so the sums are bit-identical.
__device__ __forceinline__ int icp_pixel_project(const float3& vcurr, int cols, int rows, const Intr& intr,
                                                 const Mat33& Rcurr, const float3& tcurr, const Mat33& Rprev_inv, const float3& tprev)
{
    if (isnan(vcurr.x)) return -1;
    float3 vcurr_g = add3(mul33(Rcurr, vcurr), tcurr);
    float3 vcurr_cp = mul33(Rprev_inv, sub3(vcurr_g, tprev));
    int2 ukr;
    ukr.x = __float2int_rn(vcurr_cp.x * intr.fx / vcurr_cp.z + intr.cx);
    ukr.y = __float2int_rn(vcurr_cp.y * intr.fy / vcurr_cp.z + intr.cy);
    if (ukr.x < 0 || ukr.y < 0 || ukr.x >= cols || ukr.y >= rows || vcurr_cp.z < 0) return -1;
    return ukr.y * cols + ukr.x;
}

__device__ __forceinline__ void icp_pixel_finish(const float3& vcurr, const float3& ncurr, const float3& vprev_g, const float3& nprev_g,
                                                 const Mat33& Rcurr, const float3& tcurr, const Mat33& Rprev_inv, const float3& tprev,
                                                 float dist_thres, float angle_thres, float (&sum)[32])
{
    if (isnan(vprev_g.x) || isnan(nprev_g.x) || isnan(ncurr.x)) return;
    float3 vcurr_g = add3(mul33(Rcurr, vcurr), tcurr);
    float3 ncurr_g = mul33(Rcurr, ncurr);
    float dist = norm3(sub3(vprev_g, vcurr_g));
    float sine = norm3(cross3(ncurr_g, nprev_g));
    if (!(sine < angle_thres && dist <= dist_thres)) return;
    float3 s_cp = mul33(Rprev_inv, sub3(vcurr_g, tprev));
    float3 d_cp = mul33(Rprev_inv, sub3(vprev_g, tprev));
    float3 n_cp = mul33(Rprev_inv, nprev_g);
    float3 sxn = cross3(s_cp, n_cp);
    const float row[7] = {n_cp.x, n_cp.y, n_cp.z, sxn.x, sxn.y, sxn.z, dot3(n_cp, sub3(s_cp, d_cp))};
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 7; ++b) sum[k++] += row[a] * row[b];
    sum[27] += row[6] * row[6];
    sum[28] += 1.f;
}

// The same split with the projection's intermediates handed over in registers instead of being recomputed: vcurr_g (volume frame) and
// vcurr_cp (previous camera frame; it IS s_cp of reduce.cu:268 -- the same expression).  Bit-identical sums to icp_pixel_staged.
__device__ __forceinline__ int icp_pixel_project2(const float3& vcurr, int cols, int rows, const Intr& intr,
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

__device__ __forceinline__ void icp_pixel_finish2(const float3& vcurr_g, const float3& s_cp, const float3& ncurr, const float3& vprev_g, const float3& nprev_g,
                                                  const Mat33& Rcurr, const Mat33& Rprev_inv, const float3& tprev,
                                                  float dist_thres, float angle_thres, float (&sum)[32])
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
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 7; ++b) sum[k++] += row[a] * row[b];
    sum[27] += row[6] * row[6];
    sum[28] += 1.f;
}

} // namespace kt
