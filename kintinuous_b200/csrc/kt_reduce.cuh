// kintinuous_b200 -- CTA / grid reduction of the 29 normal-equation sums (JtJJtrSE3, cuda/internal.h:98-149).
// Replaces warpReduceSum / blockReduceSum / reduceSum<<<1, MAX_THREADS>>> (cuda/reduce.cu:88-184): shuffle tree per
// warp -> shared memory -> one 128-byte partial per CTA -> the last CTA (ticket counter) sums the partials in a fixed
// order, so the result is deterministic run to run and no second launch / host sync is needed.
#pragma once
#include "kt_ops.h"

namespace kt {

enum { RED_THREADS = 256, NSUM = 29 };

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// All RED_THREADS threads of every CTA call this.  Returns true in the last CTA to finish, with the grid totals in
// s_red[0][0..28] (valid after the call for all its threads).
__device__ __forceinline__ bool grid_reduce29(float (&sum)[NSUM], float* __restrict__ partials, unsigned int* counter,
                                              float (*s_red)[32], bool* s_last)
{
    const int tid = threadIdx.x;
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int k = 0; k < NSUM; ++k) {
        float v = warp_sum(sum[k]);
        if (lane == 0) s_red[wid][k] = v;
    }
    __syncthreads();
    if (tid < NSUM) {
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < RED_THREADS / 32; ++w) v += s_red[w][tid];
        partials[blockIdx.x * 32 + tid] = v;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        unsigned int ticket = atomicInc(counter, gridDim.x - 1);      // wraps back to 0 for the next launch
        *s_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!*s_last) return false;
    __threadfence();
    {
        const int k = tid & 31, part = tid >> 5;                       // 8 interleaved partial sums per component
        float v = 0.f;
        if (k < NSUM)
            for (int b = part; b < (int)gridDim.x; b += RED_THREADS / 32) v += __ldcg(&partials[b * 32 + k]);
        s_red[part][k] = v;
    }
    __syncthreads();
    float tot = 0.f;
    if (tid < NSUM) {
#pragma unroll
        for (int w = 0; w < RED_THREADS / 32; ++w) tot += s_red[w][tid];
    }
    __syncthreads();
    if (tid < NSUM) s_red[0][tid] = tot;
    __syncthreads();
    return true;
}

// The only code that adds a row to the 29 sums (getProducts, reduce.cu:279-313).  S: NSUM, or the 32 of the whole-frame kernels,
// which transpose-reduce a full warp's worth of components.
template <int S>
__device__ __forceinline__ void accumulate_row(float (&sum)[S], const float (&row)[7])
{
    static_assert(S >= NSUM, "accumulate_row: fewer than 29 sums");
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 7; ++b) sum[k++] += row[a] * row[b];
    sum[27] += row[6] * row[6];
    sum[28] += 1.f;
}

int reduce_grid_for(int n_items);

} // namespace kt
