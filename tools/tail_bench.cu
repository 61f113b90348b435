// Micro-benchmark (development tool, not product): the per-iteration TAIL of the whole-frame odometry kernels in isolation --
// "every CTA contributes 29 floats, every CTA ends up with the 29 grid totals and the solved pose" -- in several designs, timed in SM
// cycles per iteration from CTA 0 over many iterations, one CTA of 512 threads per SM like icp_frame_kernel.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I kintinuous_b200/csrc tools/tail_bench.cu -o tools/bin/tail_bench   (tools/bin/ is git-ignored)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#include "kt_ops.h"
#include "kt_solve.cuh"
#include "kt_frame.cuh"
namespace cg = cooperative_groups;
using namespace kt;

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

enum { T = 512, NS = 29 };

struct P {
    float* partials;                 // [2][32][G]
    unsigned int* bar;               // counter
    unsigned long long* acc;         // [4][32] fixed-point accumulators
    unsigned long long* ll;          // [2][G][32] {value, tag} pairs
    unsigned long long* ll2;         // [2][64][32] second-level pairs
    long long* cycles;               // [iters] per-iteration cycles of CTA 0
    float* out;                      // [32] checksum
    int iters;
    int solve;                       // 0 none, 1 thread-0 FP64 solve as in icp_frame_kernel
};

__device__ __forceinline__ float my_value(int comp, int it) { return (float)((blockIdx.x * 31 + comp * 7 + it) % 97) * 0.125f + 1.0f; }

__device__ __forceinline__ void do_solve(const float* s_sum, double* s_Rt, float* s_Rp, float* s_tp, float* s_R, float* s_t)
{
    double dA[36], db[6];
    int shift = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = i; j < 7; ++j) {
            double value = (double)s_sum[shift++];
            if (j == 6) db[i] = value * 1e-6; else { if (i == j) value += 1e4; dA[j * 6 + i] = value; dA[i * 6 + j] = value; }
        }
    gauss_newton_update_p(dA, db, s_Rt, s_Rp, s_tp, s_R, s_t);
}
__device__ __forceinline__ void do_solve_fast(const float* s_sum, double* s_Rt, float* s_Rp, float* s_tp, float* s_R, float* s_t)
{
    double dA[36], db[6];
    int shift = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = i; j < 7; ++j) {
            double value = (double)s_sum[shift++];
            if (j == 6) db[i] = value * 1e-6; else { if (i == j) value += 1e4; dA[j * 6 + i] = value; dA[i * 6 + j] = value; }
        }
    gauss_newton_update_fast(dA, db, s_Rt, s_Rp, s_tp, s_R, s_t);
}

// counter barrier: every CTA adds 1 and spins until all G have arrived at `target` (a multiple of G)
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

// ---- V0: what icp_frame_kernel does today -------------------------------------------------------------------------------
__global__ void __launch_bounds__(T, 1) v0_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    const int tid = threadIdx.x, G = gridDim.x;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    unsigned int target = 0;
    float chk = 0.f;
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        float* part = p.partials + (size_t)(it & 1) * 32 * G;
        if (tid < NS) part[(size_t)tid * G + blockIdx.x] = my_value(tid, it) + s_t[0] * 1e-9f;
        target += G;
        grid_barrier(p.bar, target);
        {
            const int comp = tid >> 4, sub = tid & 15;
            float x[10];
#pragma unroll
            for (int q = 0; q < 10; ++q) { const int b = sub + 16 * q; x[q] = (comp < NS && b < G) ? __ldcg(&part[(size_t)comp * G + b]) : 0.f; }
            float v = 0.f;
#pragma unroll
            for (int q = 0; q < 10; ++q) v += x[q];
            v += __shfl_xor_sync(0xffffffffu, v, 8); v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
            if (sub == 0 && comp < NS) s_sum[comp] = v;
        }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}

// ---- V1: fixed-point 64-bit atomic accumulators (order-independent => deterministic) + release counter ------------------
__device__ __forceinline__ unsigned int ld_acquire(const unsigned int* p) { unsigned int v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void red_release_add(unsigned int* p, unsigned int v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }

__global__ void __launch_bounds__(T, 1) v1_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    const int tid = threadIdx.x, G = gridDim.x;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    unsigned int target = 0;
    float chk = 0.f;
    const double SCALE = 4294967296.0;           // 2^32
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        unsigned long long* acc = p.acc + (size_t)(it & 3) * 32;
        target += G;
        if (tid < 32) {
            if (tid < NS) {
                const float v = my_value(tid, it) + s_t[0] * 1e-9f;
                red_add_u64(&acc[tid], (unsigned long long)__double2ll_rn((double)v * SCALE));
            }
            if (blockIdx.x == 0) p.acc[(size_t)((it + 2) & 3) * 32 + tid] = 0ull;        // the buffer two iterations ahead (nobody touches it now)
            __syncwarp();
            if (tid == 0) {
                red_release_add(p.bar, 1u);
                while ((int)(ld_acquire(p.bar) - target) < 0) { }
            }
            __syncwarp();
            if (tid < NS) s_sum[tid] = (float)((double)(long long)ld_relaxed_u64(&acc[tid]) * (1.0 / SCALE));
        }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}

// ---- V2: flat LL exchange: every CTA writes 29 {value, tag} pairs, every CTA polls all G x 29 pairs ---------------------
__device__ __forceinline__ void st_ll(unsigned long long* p, float v, unsigned int tag)
{ asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" :: "l"(p), "r"(__float_as_uint(v)), "r"(tag) : "memory"); }
__device__ __forceinline__ bool ld_ll(const unsigned long long* p, unsigned int tag, float& v)
{ unsigned int a, b; asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "l"(p) : "memory"); v = __uint_as_float(a); return b == tag; }

__global__ void __launch_bounds__(T, 1) v2_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    __shared__ float s_part[16][32];
    const int tid = threadIdx.x, G = gridDim.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    float chk = 0.f;
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        const unsigned int tag = (unsigned int)it + 1u;
        unsigned long long* ll = p.ll + (size_t)(it & 1) * G * 32;
        if (tid < NS) st_ll(&ll[(size_t)blockIdx.x * 32 + tid], my_value(tid, it) + s_t[0] * 1e-9f, tag);
        // warp w sums CTAs w, w+16, ... in a fixed order; lane = component
        float v = 0.f;
        if (lane < NS)
            for (int b = wid; b < G; b += 16) { float x; while (!ld_ll(&ll[(size_t)b * 32 + lane], tag, x)) { } v += x; }
        s_part[wid][lane] = v;
        __syncthreads();
        if (tid < NS) { float t = 0.f;
#pragma unroll
            for (int w = 0; w < 16; ++w) t += s_part[w][tid];
            s_sum[tid] = t; }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}

// ---- V3: cluster of CS CTAs: DSMEM gather to every CTA of the cluster, one cluster barrier, then LL among cluster leaders
// (G / CS leaders x 29 pairs, polled by every CTA) ---------------------------------------------------------------------------
template <int CS>
__global__ void __launch_bounds__(T, 1) v3_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    __shared__ float s_cl[2][CS][32];          // partials of the cluster's CTAs, double-buffered by iteration parity
    __shared__ float s_part[16][32];
    cg::cluster_group cl = cg::this_cluster();
    const int tid = threadIdx.x, G = gridDim.x, lane = tid & 31, wid = tid >> 5;
    const int crank = (int)cl.block_rank(), NC = G / CS, cid = blockIdx.x / CS;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    cl.sync();
    float chk = 0.f;
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        const unsigned int tag = (unsigned int)it + 1u;
        // 1. my partial into the leader's shared memory (DSMEM store), cluster barrier
        if (tid < NS) {
            float* dst = cl.map_shared_rank(&s_cl[it & 1][crank][tid], 0);
            *dst = my_value(tid, it) + s_t[0] * 1e-9f;
        }
        cl.sync();
        unsigned long long* ll = p.ll + (size_t)(it & 1) * G * 32;
        if (crank == 0 && tid < NS) {
            float v = 0.f;
#pragma unroll
            for (int c = 0; c < CS; ++c) v += s_cl[it & 1][c][tid];
            st_ll(&ll[(size_t)cid * 32 + tid], v, tag);
        }
        float v = 0.f;
        if (lane < NS)
            for (int b = wid; b < NC; b += 16) { float x; while (!ld_ll(&ll[(size_t)b * 32 + lane], tag, x)) { } v += x; }
        s_part[wid][lane] = v;
        __syncthreads();
        if (tid < NS) { float t = 0.f;
#pragma unroll
            for (int w = 0; w < 16; ++w) t += s_part[w][tid];
            s_sum[tid] = t; }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}

// ---- V4: two-level LL without clusters: CTA b writes pairs; NR reducer CTAs (b % (G/NR) == 0) each sum their group's pairs and
// publish a second-level pair set; everybody polls the NR x 29 second-level pairs --------------------------------------------
template <int NR>
__global__ void __launch_bounds__(T, 1) v4_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    __shared__ float s_part[16][32];
    const int tid = threadIdx.x, G = gridDim.x, lane = tid & 31, wid = tid >> 5;
    const int GS = (G + NR - 1) / NR, grp = blockIdx.x / GS; const bool reducer = (blockIdx.x % GS) == 0;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    float chk = 0.f;
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        const unsigned int tag = (unsigned int)it + 1u;
        unsigned long long* ll = p.ll + (size_t)(it & 1) * G * 32;
        unsigned long long* ll2 = p.ll2 + (size_t)(it & 1) * 64 * 32;
        if (tid < NS) st_ll(&ll[(size_t)blockIdx.x * 32 + tid], my_value(tid, it) + s_t[0] * 1e-9f, tag);
        if (reducer) {
            const int b0 = grp * GS, b1 = min(G, b0 + GS);
            float v = 0.f;
            if (lane < NS)
                for (int b = b0 + wid; b < b1; b += 16) { float x; while (!ld_ll(&ll[(size_t)b * 32 + lane], tag, x)) { } v += x; }
            s_part[wid][lane] = v;
            __syncthreads();
            if (tid < NS) { float t = 0.f;
#pragma unroll
                for (int w = 0; w < 16; ++w) t += s_part[w][tid];
                st_ll(&ll2[(size_t)grp * 32 + tid], t, tag); }
        }
        if (tid < 32) {
            float t = 0.f;
            if (lane < NS)
                for (int g = 0; g < NR; ++g) { float x; while (!ld_ll(&ll2[(size_t)g * 32 + lane], tag, x)) { } t += x; }
            if (lane < NS) s_sum[lane] = t;
        }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}

// ---- V5: like V0 but the barrier is release/acquire PTX instead of __threadfence + atomicAdd + volatile poll + __threadfence --
__global__ void __launch_bounds__(T, 1) v5_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    const int tid = threadIdx.x, G = gridDim.x;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    unsigned int target = 0;
    float chk = 0.f;
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        float* part = p.partials + (size_t)(it & 1) * 32 * G;
        target += G;
        if (tid < 32) {
            if (tid < NS) part[(size_t)tid * G + blockIdx.x] = my_value(tid, it) + s_t[0] * 1e-9f;
            __syncwarp();
            if (tid == 0) { red_release_add(p.bar, 1u); while ((int)(ld_acquire(p.bar) - target) < 0) { } }
        }
        __syncthreads();
        {
            const int comp = tid >> 4, sub = tid & 15;
            float x[10];
#pragma unroll
            for (int q = 0; q < 10; ++q) { const int b = sub + 16 * q; x[q] = (comp < NS && b < G) ? __ldcg(&part[(size_t)comp * G + b]) : 0.f; }
            float v = 0.f;
#pragma unroll
            for (int q = 0; q < 10; ++q) v += x[q];
            v += __shfl_xor_sync(0xffffffffu, v, 8); v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 2); v += __shfl_xor_sync(0xffffffffu, v, 1);
            if (sub == 0 && comp < NS) s_sum[comp] = v;
        }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}


// ---- V6: self-counting fixed-point words.  Every CTA adds (fixed-point value with the low 8 bits cleared) + 1 to 29 64-bit words; the
// low byte of (word_now - word_at_the_previous_use) therefore counts arrivals and the rest is the exact integer sum: no counter, no
// fence, no zeroing (two word sets by iteration parity, persistent).  STRIDE = distance between the 29 words in 8-byte units. --------
template <int STRIDE, int FASTSOLVE>
__global__ void __launch_bounds__(T, 1) v6_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    const int tid = threadIdx.x, G = gridDim.x;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    float chk = 0.f;
    unsigned long long prev[2] = {0ull, 0ull};
    unsigned long long* w0 = p.ll;                                   // [2][32 * STRIDE]
    if (tid < NS) { prev[0] = ld_relaxed_u64(&w0[(size_t)tid * STRIDE]); prev[1] = ld_relaxed_u64(&w0[(size_t)(32 + tid) * STRIDE]); }
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        if (tid < 32) {
            unsigned long long* w = w0 + (size_t)(it & 1) * 32 * STRIDE + (size_t)tid * STRIDE;
            if (tid < NS) {
                const float v = my_value(tid, it) + s_t[0] * 1e-9f;
                const long long q = __double2ll_rn((double)v * 4294967296.0) & ~0xFFll;
                red_add_u64(w, (unsigned long long)(q + 1));
                unsigned long long now, d;
                do { now = ld_relaxed_u64(w); d = now - prev[it & 1]; } while ((unsigned int)(d & 0xFFull) != (unsigned int)G);
                prev[it & 1] = now;
                s_sum[tid] = (float)((double)(long long)(d - (unsigned long long)G) * (1.0 / 4294967296.0));
            }
        }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}

// ---- V7: the exchanges the odometry kernels use (kt_frame.cuh, words XW_STRIDE apart): grid_sum_words, one word per component, against
// grid_sum_words_wide, two (the photometric sums of rgbd_frame_kernel, whose range one word cannot hold). -------------------------------
template <int WIDE>
__global__ void __launch_bounds__(T, 1) v7_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    const int tid = threadIdx.x, G = gridDim.x;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    __syncthreads();
    float chk = 0.f;
    GridSumState st; st.prev[0] = 0ull; st.prev[1] = 0ull;
    GridSumState st_lo = st;
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        if (tid < 32) {
            const float v = tid < NS ? my_value(tid, it) + s_t[0] * 1e-9f : 0.f;
            const double tot = WIDE ? grid_sum_words_wide(p.ll, it, tid, v, st, st_lo, (unsigned int)G, nullptr)
                                    : grid_sum_words(p.ll, it, tid, v, st, (unsigned int)G, nullptr);
            if (tid < NS) s_sum[tid] = (float)tot;
        }
        __syncthreads();
        if (tid == 0 && p.solve) do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t);
        __syncthreads();
        chk += s_sum[5] + s_t[1];
        if (blockIdx.x == 0 && tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0 && blockIdx.x == 0) p.out[0] = chk;
}

// ---- the solve alone, on one thread of one CTA, sums in shared memory ---------------------------------------------------
template <int FAST> __global__ void solve_only_kernel(P p)
{
    __shared__ float s_sum[32]; __shared__ double s_Rt[16]; __shared__ float s_Rp[9], s_tp[3], s_R[9], s_t[3];
    const int tid = threadIdx.x;
    if (tid == 0) { for (int k = 0; k < 16; ++k) s_Rt[k] = (k % 5 == 0); for (int k = 0; k < 9; ++k) { s_Rp[k] = (k % 4 == 0); s_R[k] = s_Rp[k]; } for (int k = 0; k < 3; ++k) { s_tp[k] = 3.f; s_t[k] = 3.f; } }
    if (tid < 32) s_sum[tid] = 1.f + tid;
    __syncthreads();
    for (int it = 0; it < p.iters; ++it) {
        long long t0 = clock64();
        if (tid == 0) { if (FAST) do_solve_fast(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t); else do_solve(s_sum, s_Rt, s_Rp, s_tp, s_R, s_t); }
        __syncthreads();
        if (tid < NS) s_sum[tid] += s_t[tid % 3] * 1e-3f;
        __syncthreads();
        if (tid == 0) p.cycles[it] = clock64() - t0;
    }
    if (tid == 0) p.out[0] = s_t[0] + s_R[1];
}

// accuracy of the device-only reciprocal path: x from ldlt6_solve_fast vs ldlt6_solve on the same systems
__global__ void solve_check_kernel(const double* A, const double* b, int n, double* maxrel)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double x0[6], x1[6];
    ldlt6_solve(A + (size_t)i * 36, b + (size_t)i * 6, x0);
    ldlt6_solve_fast(A + (size_t)i * 36, b + (size_t)i * 6, x1);
    double num = 0, den = 1e-300;
    for (int k = 0; k < 6; ++k) { num = fmax(num, fabs(x0[k] - x1[k])); den = fmax(den, fabs(x0[k])); }
    maxrel[i] = num / den;
}

template <class K> static void run(const char* name, K kernel, P p, int grid, int cluster, bool coop)
{
    CK(cudaMemset(p.bar, 0, 4)); CK(cudaMemset(p.acc, 0, 4 * 32 * 8)); CK(cudaMemset(p.ll, 0, (size_t)2 * 4096 * 32 * 8)); CK(cudaMemset(p.ll2, 0, (size_t)2 * 64 * 32 * 8));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    cudaLaunchConfig_t cfg; memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(T); cfg.dynamicSmemBytes = 0; cfg.stream = 0;
    cudaLaunchAttribute at[2]; int na = 0;
    if (coop) { at[na].id = cudaLaunchAttributeCooperative; at[na].val.cooperative = 1; ++na; }
    if (cluster > 1) { at[na].id = cudaLaunchAttributeClusterDimension; at[na].val.clusterDim.x = cluster; at[na].val.clusterDim.y = 1; at[na].val.clusterDim.z = 1; ++na; }
    cfg.attrs = at; cfg.numAttrs = na;
    if (cluster > 8) CK(cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    CK(cudaEventRecord(e0));
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, p);
    if (e != cudaSuccess) { printf("%-44s launch failed: %s\n", name, cudaGetErrorString(e)); cudaGetLastError(); return; }
    CK(cudaEventRecord(e1));
    CK(cudaDeviceSynchronize());
    float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
    std::vector<long long> cyc(p.iters);
    CK(cudaMemcpy(cyc.data(), p.cycles, p.iters * sizeof(long long), cudaMemcpyDeviceToHost));
    double mean = 0; long long mn = 1LL << 60; for (int i = 50; i < p.iters; ++i) { mean += cyc[i]; if (cyc[i] < mn) mn = cyc[i]; } mean /= (p.iters - 50);
    printf("%-44s grid %3d  cycles/iter mean %7.0f min %6lld   us/iter %.3f\n", name, grid, mean, mn, ms * 1e3 / p.iters);
}

int main()
{
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    P p; p.iters = 2000;
    CK(cudaMalloc(&p.partials, 2 * 32 * 1024 * 4)); CK(cudaMalloc(&p.bar, 4)); CK(cudaMalloc(&p.acc, 4 * 32 * 8));
    CK(cudaMalloc(&p.ll, (size_t)2 * 4096 * 32 * 8)); CK(cudaMalloc(&p.ll2, (size_t)2 * 64 * 32 * 8));
    CK(cudaMalloc(&p.cycles, p.iters * 8)); CK(cudaMalloc(&p.out, 128));
    printf("SMs %d\n", sms);
    for (int solve = 0; solve < 2; ++solve) {
        p.solve = solve;
        printf("---- solve %d ----\n", solve);
        run("V0 partials + fence/atomic barrier (today)", v0_kernel, p, sms, 1, true);
        run("V5 partials + release/acquire barrier", v5_kernel, p, sms, 1, true);
        run("V1 fixed-point red.u64 + release counter", v1_kernel, p, sms, 1, true);
        run("V2 flat LL (every CTA polls all)", v2_kernel, p, sms, 1, true);
        run("V3 cluster 2 DSMEM + LL leaders", v3_kernel<2>, p, sms, 2, true);
        run("V3 cluster 4 DSMEM + LL leaders", v3_kernel<4>, p, sms, 4, true);
        run("V3 cluster 8 DSMEM + LL leaders", v3_kernel<8>, p, 144, 8, true);
        run("V3 cluster 16 DSMEM + LL leaders", v3_kernel<16>, p, 128, 16, true);
        run("V6 self-counting words, packed", v6_kernel<1, 0>, p, sms, 1, true);
        run("V6 self-counting words, stride 256 B", v6_kernel<32, 0>, p, sms, 1, true);
        run("V6 self-counting words, stride 1280 B", v6_kernel<160, 0>, p, sms, 1, true);
        run("V6 self-counting words, stride 2304 B", v6_kernel<288, 0>, p, sms, 1, true);
        run("V6 self-counting words, stride 4352 B", v6_kernel<544, 0>, p, sms, 1, true);
        run("V6 self-counting words, stride 5376 B", v6_kernel<672, 0>, p, sms, 1, true);
        run("V6 self-counting words, stride 16640 B", v6_kernel<2080, 0>, p, sms, 1, true);
        run("V6 stride 256 B, 16 CTAs", v6_kernel<32, 0>, p, 16, 1, true);
        run("V6 stride 256 B, 32 CTAs", v6_kernel<32, 0>, p, 32, 1, true);
        run("V6 stride 256 B, 74 CTAs", v6_kernel<32, 0>, p, 74, 1, true);
        run("V7 grid_sum_words (one word)", v7_kernel<0>, p, sms, 1, true);
        run("V7 grid_sum_words_wide (two words)", v7_kernel<1>, p, sms, 1, true);
        run("V4 two-level LL, 4 reducers", v4_kernel<4>, p, sms, 1, true);
        run("V4 two-level LL, 8 reducers", v4_kernel<8>, p, sms, 1, true);
        run("V4 two-level LL, 12 reducers", v4_kernel<12>, p, sms, 1, true);
        // small grids (what one cluster would replace at the coarse levels)
        run("V3 ONE cluster of 8", v3_kernel<8>, p, 8, 8, false);
        run("V3 ONE cluster of 16", v3_kernel<16>, p, 16, 16, false);
        run("V2 flat LL, 16 CTAs", v2_kernel, p, 16, 1, true);
        run("V2 flat LL, 37 CTAs", v2_kernel, p, 37, 1, true);
    }
    {
        const int n = 4096;
        std::vector<double> hA((size_t)n * 36), hb((size_t)n * 6), hr(n);
        srand(7);
        for (int i = 0; i < n; ++i) {
            double J[40][6];
            const double sc = (i % 3 == 0) ? 300.0 : (i % 3 == 1 ? 1.0 : 1e-2);
            for (int r = 0; r < 40; ++r) for (int c = 0; c < 6; ++c) J[r][c] = sc * ((rand() / (double)RAND_MAX) - 0.5) * (c < 3 ? 1.0 : 0.3);
            for (int a = 0; a < 6; ++a) for (int c = 0; c < 6; ++c) { double s = 0; for (int r = 0; r < 40; ++r) s += J[r][a] * J[r][c]; hA[(size_t)i * 36 + a * 6 + c] = s; }
            for (int c = 0; c < 6; ++c) hb[(size_t)i * 6 + c] = (rand() / (double)RAND_MAX) - 0.5;
        }
        double *dA, *db, *dr; CK(cudaMalloc(&dA, hA.size() * 8)); CK(cudaMalloc(&db, hb.size() * 8)); CK(cudaMalloc(&dr, n * 8));
        CK(cudaMemcpy(dA, hA.data(), hA.size() * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(db, hb.data(), hb.size() * 8, cudaMemcpyHostToDevice));
        solve_check_kernel<<<(n + 127) / 128, 128>>>(dA, db, n, dr); CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(hr.data(), dr, n * 8, cudaMemcpyDeviceToHost));
        double w = 0; for (int i = 0; i < n; ++i) w = hr[i] > w ? hr[i] : w;
        printf("ldlt6_solve_fast vs ldlt6_solve on %d random SPD systems: max relative difference of x = %.3e\n", n, w);
    }
    run("solve only (thread 0, sums in smem)", solve_only_kernel<0>, p, 1, 1, false);
    run("solve only, trimmed (rcp+Newton, series Rodrigues)", solve_only_kernel<1>, p, 1, 1, false);
    return 0;
}
