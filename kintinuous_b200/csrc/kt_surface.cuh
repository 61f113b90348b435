// kintinuous_b200 -- the zero-crossing arithmetic shared by the point extraction (kt_extract.cu) and the mesher (kt_mesh.cu), so that a
// mesh vertex and the extracted point of the same edge are the same bits.
#pragma once
#include "kt_common.cuh"

namespace kt {

// a voxel takes part in a surface when it has been observed and is not at the positive truncation limit (extract.cu:139-150)
__device__ __forceinline__ bool surface_voxel(int W, float F) { return W != 0 && F != 1.f; }

// (V * |Fn| + Vn * |F|) * d_inv with the contraction the reference build has (extract.cu:155, checked in its SASS:
// FMUL V*|Fn|; FFMA |F|*Vn + that; FMUL by the reciprocal).  Left to the compiler, the choice of which product is fused
// changes with unrelated edits and moves the point by 1 ulp.
__device__ __forceinline__ float interp(float V, float Vn, float F, float Fn, float d_inv)
{
    return __fmul_rn(__fmaf_rn(fabsf(F), Vn, __fmul_rn(V, fabsf(Fn))), d_inv);
}

// volume coordinate (metres from the volume corner) -> slice coordinate: realVoxelWrap * cell - size / 2 (extract.cu:310-312)
__device__ __forceinline__ float slice_coord(float v, int real_wrap, float cell, int V)
{
    return v + real_wrap * cell - ((cell * V) / 2);
}

} // namespace kt
