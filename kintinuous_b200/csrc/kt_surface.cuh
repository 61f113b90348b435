// kintinuous_b200 -- the zero-crossing arithmetic shared by the point extraction (kt_extract.cu) and the meshers (kt_mesh.cu,
// kt_mapvol.cu), so that a mesh vertex and the extracted point of the same edge are the same bits.
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

// ---- marching cubes over a field: the per-voxel half of kt_mesh.cu's contract, shared by the dense box (kt_mesh.cu) and the brick set
// of the global map (kt_mapvol.cu).  A Field answers, for voxel (x, y, z) of its lattice:
//   bool corner(x, y, z, short& raw)   a valid corner (surface_voxel, W >= the cull; raw set when it is);
//   short raw(x, y, z), uchar4 color(x, y, z)   for a voxel that is one.

const unsigned int MC_CELL_CORNERS = 0x361Bu;   // bits of the 8 corners of a cell in a 3x3x3 neighbourhood (index dx + 3 dy + 9 dz), cell at 0

// What voxel (x, y, z) owns: the crossing edges a meshed cell uses (vflags bit a = axis a) and, when cell (x, y, z) is meshed, its case
// (else -1).  cell_allowed(cx, cy, cz): whether the field may mesh the cell whose lower corner is (cx, cy, cz) at all (box, border).
struct McVoxel { unsigned int vflags; int mc_case; };

template <class Field, class Allowed>
__device__ __forceinline__ McVoxel mc_classify(const Field& f, int x, int y, int z, const Allowed& cell_allowed)
{
    McVoxel v; v.vflags = 0; v.mc_case = -1;
    short r;
    if (!f.corner(x, y, z, r)) return v;                  // an invalid voxel is no cell's corner and owns no edge
    unsigned int valid = 0, inside = 0;
#pragma unroll
    for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int b = (dx + 1) + 3 * (dy + 1) + 9 * (dz + 1);
                short q;
                if (f.corner(x + dx, y + dy, z + dz, q)) { valid |= 1u << b; if (q < 0) inside |= 1u << b; }
            }
    // cell whose lower corner is (x + ox, y + oy, z + oz), o in {-1, 0}^3: allowed and 8 valid corners
    auto cell_ok = [&](int ox, int oy, int oz) -> bool {
        if (!cell_allowed(x + ox, y + oy, z + oz)) return false;
        const unsigned int m = MC_CELL_CORNERS << ((ox + 1) + 3 * (oy + 1) + 9 * (oz + 1));
        return (valid & m) == m;
    };
    if (cell_ok(0, 0, 0)) {
        int c = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) c |= (int)((inside >> (13 + (k & 1) + 3 * ((k >> 1) & 1) + 9 * (k >> 2))) & 1u) << k;
        if (c != 0 && c != 255) v.mc_case = c;
    }
    const bool in0 = (inside >> 13) & 1u;
    // x edge: (x, y, z) - (x + 1, y, z), used by the cells at (x, y - dy, z - dz)
    if (((valid >> 14) & 1u) && (((inside >> 14) & 1u) != in0) &&
        (cell_ok(0, 0, 0) || cell_ok(0, -1, 0) || cell_ok(0, 0, -1) || cell_ok(0, -1, -1))) v.vflags |= 1u;
    if (((valid >> 16) & 1u) && (((inside >> 16) & 1u) != in0) &&
        (cell_ok(0, 0, 0) || cell_ok(-1, 0, 0) || cell_ok(0, 0, -1) || cell_ok(-1, 0, -1))) v.vflags |= 2u;
    if (((valid >> 22) & 1u) && (((inside >> 22) & 1u) != in0) &&
        (cell_ok(0, 0, 0) || cell_ok(-1, 0, 0) || cell_ok(0, -1, 0) || cell_ok(-1, -1, 0))) v.vflags |= 4u;
    return v;
}

// TSDF gradient at a valid voxel (raw r0), per metre, in raw units: central differences, one-sided next to an invalid voxel, 0 if neither
// neighbour is valid
template <class Field>
__device__ __forceinline__ float3 mc_gradient(const Field& f, const float3& inv_cell, int x, int y, int z, short r0)
{
    float g[3];
    const float inv[3] = {inv_cell.x, inv_cell.y, inv_cell.z};
#pragma unroll
    for (int b = 0; b < 3; ++b) {
        const int dx = b == 0, dy = b == 1, dz = b == 2;
        short rm = 0, rp = 0;
        const bool okm = f.corner(x - dx, y - dy, z - dz, rm), okp = f.corner(x + dx, y + dy, z + dz, rp);
        g[b] = okm && okp ? (float)(rp - rm) * 0.5f * inv[b] : okp ? (float)(rp - r0) * inv[b] : okm ? (float)(r0 - rm) * inv[b] : 0.f;
    }
    return make_float3(g[0], g[1], g[2]);
}

// The 32-byte kt_mesh_vertex of the edge (x, y, z) - (x, y, z) + e_a: extract_kernel's point, the blended gradient normal, the colour
// of the end nearer the surface.  V and real_wrap place the lattice as slice_coord does.
template <class Field>
__device__ __forceinline__ void mc_vertex(const Field& f, const float3& cell, const float3& inv_cell, const int3& real_wrap, int V,
                                          int x, int y, int z, int a, uint4* out)
{
    const int dx = a == 0, dy = a == 1, dz = a == 2;
    const short r0 = f.raw(x, y, z), r1 = f.raw(x + dx, y + dy, z + dz);
    const float F = unpack_tsdf(r0), Fn = unpack_tsdf(r1);
    // extract_kernel's point for this edge (kt_extract.cu), expression for expression
    float3 Vc;
    Vc.x = (x + 0.5f) * cell.x; Vc.y = (y + 0.5f) * cell.y; Vc.z = (z + 0.5f) * cell.z;
    const float d_inv = 1.f / (fabs(F) + fabs(Fn));
    if (a == 0) { float Vnx = Vc.x + cell.x; Vc.x = interp(Vc.x, Vnx, F, Fn, d_inv); }
    else if (a == 1) { float Vny = Vc.y + cell.y; Vc.y = interp(Vc.y, Vny, F, Fn, d_inv); }
    else { float Vnz = Vc.z + cell.z; Vc.z = interp(Vc.z, Vnz, F, Fn, d_inv); }
    const float px = slice_coord(Vc.x, real_wrap.x, cell.x, V);
    const float py = slice_coord(Vc.y, real_wrap.y, cell.y, V);
    const float pz = slice_coord(Vc.z, real_wrap.z, cell.z, V);
    const float3 g0 = mc_gradient(f, inv_cell, x, y, z, r0), g1 = mc_gradient(f, inv_cell, x + dx, y + dy, z + dz, r1);
    const float w0 = fabsf(Fn) * d_inv, w1 = fabsf(F) * d_inv;
    float3 n = make_float3(w0 * g0.x + w1 * g1.x, w0 * g0.y + w1 * g1.y, w0 * g0.z + w1 * g1.z);
    const float l2 = n.x * n.x + n.y * n.y + n.z * n.z;
    if (l2 > 0.f) { const float s = rsqrtf(l2); n.x *= s; n.y *= s; n.z *= s; } else n = make_float3(0.f, 0.f, 0.f);
    const bool lower = abs((int)r0) <= abs((int)r1);
    const uchar4 c = lower ? f.color(x, y, z) : f.color(x + dx, y + dy, z + dz);
    const unsigned int rgba = (unsigned int)c.z | ((unsigned int)c.y << 8) | ((unsigned int)c.x << 16) | ((unsigned int)c.w << 24);
    out[0] = make_uint4(__float_as_uint(px), __float_as_uint(py), __float_as_uint(pz), __float_as_uint(n.x));
    out[1] = make_uint4(__float_as_uint(n.y), __float_as_uint(n.z), rgba, 0u);
}

} // namespace kt
