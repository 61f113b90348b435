// kintinuous_b200 -- marching cubes over a box of the cyclic TSDF volume: an indexed triangle mesh of the surface.
//
// Stands in for (reference, src/backend/MeshGenerator.cpp:193-227): MeshGenerator::calculateMesh, PCL's greedy projection triangulation
// of every slice's processed cloud on the CPU.  This is a different algorithm (marching cubes on the TSDF the slice is cut from, while
// it is still on the device), so there is no parity with PCL; what is kept is the input (the voxels the weight-culled processed cloud
// comes from) and the positions (each vertex is exactly the point extract_kernel emits for its edge, kt_surface.cuh).
//
// Contract (restated in numpy by the test-side mesh_oracle.py):
//   * corner valid: surface_voxel(W, F) (extract_kernel's test) and W >= weight_cull; inside: raw < 0;
//   * cell (x, y, z) = the cube whose lower corner is voxel (x, y, z); meshed when that corner is in the box, x + 1, y + 1, z + 1 < V
//     (no cyclic wrap), its 8 corners are valid and not all on the same side;
//   * one vertex per crossing edge used by a meshed cell, owned by the edge's lower voxel; vertices ordered by owner in logical order
//     (x fastest) then edge axis; triangles (kt_mc_table.h) ordered by cell in logical order, then table order;
//   * normal: TSDF gradient (central differences, one-sided at the volume border or next to an invalid voxel, 0 if neither neighbour is
//     usable) at both ends of the edge, blended with the position's weights, normalised ((0, 0, 0) when degenerate); colour: the end
//     with the smaller |raw| (ties: the lower end), r = colour.z, b = colour.x as in extract (Q8), alpha = that voxel's weight.
// Design: the work runs over the OWNER grid [minX, min(maxX + 1, V)) x ... in fixed tiles of MESH_TILE consecutive voxels (logical
// order), so block order is output order.  Count (per-tile vertex / triangle totals) -> CUB exclusive scan of the tile totals ->
// vertex pass (block scan inside the tile; each vertex also writes its key 3 * owner + axis, ascending by construction) -> triangle
// pass (keys of a cell's edges found by binary search in the key array; optionally each triangle's cell as its owner-grid index).  No atomics, so the output does not depend on the launch;
// scratch is 32 B per tile + 8 B per vertex + CUB's temporary storage.  Every pass re-derives a voxel's 3x3x3 neighbourhood from
// the volume (L1 / L2 resident) instead of storing per-cell flags.
#include "kt_ops.h"
#include "kt_surface.cuh"
#include "../../include/kintinuous_b200.h"
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>
#define KT_MC_STORAGE static __device__ const
#include "kt_mc_table.h"

namespace kt {

namespace {

const int MESH_THREADS = 256;
const int MESH_ITEMS = 16;
const long long MESH_TILE = (long long)MESH_THREADS * MESH_ITEMS;
const unsigned int CELL_CORNERS = 0x361Bu;     // bits of the 8 corners of a cell in a 3x3x3 neighbourhood (index dx + 3 dy + 9 dz), cell at 0

struct MeshParams {
    const int16_t* tsdf; const uchar4* color; int V; int3 wrap; int3 real_wrap; float3 cell, inv_cell; int cull;
    int minX, maxX, minY, maxY, minZ, maxZ;
    int ex, ey;                    // owner grid extents in x, y; its origin is (minX, minY, minZ)
    long long total;               // owner grid voxels
};

__device__ __forceinline__ int wrap1(int v, int w, int V) { v += w; return v >= V ? v - V : v; }
__device__ __forceinline__ size_t vaddr(const MeshParams& p, int x, int y, int z)
{
    return ((size_t)wrap1(z, p.wrap.z, p.V) * p.V + wrap1(y, p.wrap.y, p.V)) * p.V + wrap1(x, p.wrap.x, p.V);
}

// logical voxel (x, y, z): inside [0, V)^3 and a valid corner?  raw is set when it is.
__device__ __forceinline__ bool corner(const MeshParams& p, int x, int y, int z, short& raw)
{
    if ((unsigned)x >= (unsigned)p.V || (unsigned)y >= (unsigned)p.V || (unsigned)z >= (unsigned)p.V) return false;
    const size_t a = vaddr(p, x, y, z);
    raw = __ldg(&p.tsdf[a]);
    const int W = __ldg(&p.color[a]).w;
    return surface_voxel(W, unpack_tsdf(raw)) && W >= p.cull;
}

__device__ __forceinline__ void owner_xyz(const MeshParams& p, long long idx, int& x, int& y, int& z)
{
    x = p.minX + (int)(idx % p.ex);
    const long long r = idx / p.ex;
    y = p.minY + (int)(r % p.ey);
    z = p.minZ + (int)(r / p.ey);
}

// What the owner voxel idx contributes: the crossing edges it owns that a meshed cell uses (bit a = axis a) and, when cell (x, y, z)
// is meshed, its case (else -1).
struct Voxel { int x, y, z; unsigned int vflags; int mc_case; };

__device__ __forceinline__ Voxel classify(const MeshParams& p, long long idx)
{
    Voxel v; owner_xyz(p, idx, v.x, v.y, v.z); v.vflags = 0; v.mc_case = -1;
    short r;
    if (!corner(p, v.x, v.y, v.z, r)) return v;           // an invalid voxel is no cell's corner and owns no edge
    unsigned int valid = 0, inside = 0;
#pragma unroll
    for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int b = (dx + 1) + 3 * (dy + 1) + 9 * (dz + 1);
                short q;
                if (corner(p, v.x + dx, v.y + dy, v.z + dz, q)) { valid |= 1u << b; if (q < 0) inside |= 1u << b; }
            }
    // cell whose lower corner is (x + ox, y + oy, z + oz), o in {-1, 0}^3: in the box, inside [0, V - 1), 8 valid corners
    auto cell_ok = [&](int ox, int oy, int oz) -> bool {
        const int cx = v.x + ox, cy = v.y + oy, cz = v.z + oz;
        if (cx < p.minX || cx >= p.maxX || cy < p.minY || cy >= p.maxY || cz < p.minZ || cz >= p.maxZ) return false;
        if (cx + 1 >= p.V || cy + 1 >= p.V || cz + 1 >= p.V) return false;
        const unsigned int m = CELL_CORNERS << ((ox + 1) + 3 * (oy + 1) + 9 * (oz + 1));
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

__device__ __forceinline__ int tri_count(const Voxel& v) { return v.mc_case < 0 ? 0 : kt_mc_tri_count[v.mc_case]; }

// per-tile totals; tile `gridDim.x` (one past the last) gets 0 so that the exclusive scan of gridDim.x + 1 entries ends in the total
__global__ void __launch_bounds__(MESH_THREADS)
mesh_count_kernel(const MeshParams p, unsigned long long* vcount, unsigned long long* tcount)
{
    typedef cub::BlockReduce<int, MESH_THREADS> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const long long base = (long long)blockIdx.x * MESH_TILE;
    int nv = 0, nt = 0;
    for (int it = 0; it < MESH_ITEMS; ++it) {
        const long long idx = base + it * MESH_THREADS + threadIdx.x;
        if (idx < p.total) { const Voxel v = classify(p, idx); nv += __popc(v.vflags); nt += tri_count(v); }
    }
    const int sv = Reduce(tmp).Sum(nv);
    __syncthreads();
    const int st = Reduce(tmp).Sum(nt);
    if (threadIdx.x == 0) {
        vcount[blockIdx.x] = (unsigned long long)sv; tcount[blockIdx.x] = (unsigned long long)st;
        if (blockIdx.x == 0) { vcount[gridDim.x] = 0; tcount[gridDim.x] = 0; }
    }
}

// TSDF gradient at a valid voxel (raw r0), per metre, in raw units
__device__ __forceinline__ float3 gradient(const MeshParams& p, int x, int y, int z, short r0)
{
    float g[3];
    const float inv[3] = {p.inv_cell.x, p.inv_cell.y, p.inv_cell.z};
#pragma unroll
    for (int b = 0; b < 3; ++b) {
        const int dx = b == 0, dy = b == 1, dz = b == 2;
        short rm = 0, rp = 0;
        const bool okm = corner(p, x - dx, y - dy, z - dz, rm), okp = corner(p, x + dx, y + dy, z + dz, rp);
        g[b] = okm && okp ? (float)(rp - rm) * 0.5f * inv[b] : okp ? (float)(rp - r0) * inv[b] : okm ? (float)(r0 - rm) * inv[b] : 0.f;
    }
    return make_float3(g[0], g[1], g[2]);
}

__device__ __forceinline__ void write_vertex(const MeshParams& p, int x, int y, int z, int a, uint4* out)
{
    const int dx = a == 0, dy = a == 1, dz = a == 2;
    const size_t a0 = vaddr(p, x, y, z), a1 = vaddr(p, x + dx, y + dy, z + dz);
    const short r0 = __ldg(&p.tsdf[a0]), r1 = __ldg(&p.tsdf[a1]);
    const float F = unpack_tsdf(r0), Fn = unpack_tsdf(r1);
    // extract_kernel's point for this edge (kt_extract.cu), expression for expression
    float3 Vc;
    Vc.x = (x + 0.5f) * p.cell.x; Vc.y = (y + 0.5f) * p.cell.y; Vc.z = (z + 0.5f) * p.cell.z;
    const float d_inv = 1.f / (fabs(F) + fabs(Fn));
    if (a == 0) { float Vnx = Vc.x + p.cell.x; Vc.x = interp(Vc.x, Vnx, F, Fn, d_inv); }
    else if (a == 1) { float Vny = Vc.y + p.cell.y; Vc.y = interp(Vc.y, Vny, F, Fn, d_inv); }
    else { float Vnz = Vc.z + p.cell.z; Vc.z = interp(Vc.z, Vnz, F, Fn, d_inv); }
    const float px = slice_coord(Vc.x, p.real_wrap.x, p.cell.x, p.V);
    const float py = slice_coord(Vc.y, p.real_wrap.y, p.cell.y, p.V);
    const float pz = slice_coord(Vc.z, p.real_wrap.z, p.cell.z, p.V);
    const float3 g0 = gradient(p, x, y, z, r0), g1 = gradient(p, x + dx, y + dy, z + dz, r1);
    const float w0 = fabsf(Fn) * d_inv, w1 = fabsf(F) * d_inv;
    float3 n = make_float3(w0 * g0.x + w1 * g1.x, w0 * g0.y + w1 * g1.y, w0 * g0.z + w1 * g1.z);
    const float l2 = n.x * n.x + n.y * n.y + n.z * n.z;
    if (l2 > 0.f) { const float s = rsqrtf(l2); n.x *= s; n.y *= s; n.z *= s; } else n = make_float3(0.f, 0.f, 0.f);
    const bool lower = abs((int)r0) <= abs((int)r1);
    const uchar4 c = __ldg(&p.color[lower ? a0 : a1]);
    const unsigned int rgba = (unsigned int)c.z | ((unsigned int)c.y << 8) | ((unsigned int)c.x << 16) | ((unsigned int)c.w << 24);
    out[0] = make_uint4(__float_as_uint(px), __float_as_uint(py), __float_as_uint(pz), __float_as_uint(n.x));
    out[1] = make_uint4(__float_as_uint(n.y), __float_as_uint(n.z), rgba, 0u);
}

__global__ void __launch_bounds__(MESH_THREADS)
mesh_vertex_kernel(const MeshParams p, const unsigned long long* voff, uint4* verts, unsigned long long* keys)
{
    typedef cub::BlockScan<int, MESH_THREADS> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const long long tile = (long long)blockIdx.x * MESH_TILE;
    unsigned long long base = voff[blockIdx.x];
    for (int it = 0; it < MESH_ITEMS; ++it) {
        const long long idx = tile + it * MESH_THREADS + threadIdx.x;
        Voxel v; v.vflags = 0;
        if (idx < p.total) v = classify(p, idx);
        int off, agg;
        Scan(tmp).ExclusiveSum(__popc(v.vflags), off, agg);
        unsigned long long slot = base + (unsigned long long)off;
        for (int a = 0; a < 3; ++a)
            if (v.vflags & (1u << a)) {
                write_vertex(p, v.x, v.y, v.z, a, verts + 2 * slot);
                keys[slot] = 3ull * (unsigned long long)idx + (unsigned long long)a;
                ++slot;
            }
        base += (unsigned long long)agg;
        __syncthreads();
    }
}

__device__ __forceinline__ unsigned int find_vertex(const unsigned long long* keys, unsigned long long n, unsigned long long key)
{
    unsigned long long lo = 0, hi = n;                   // first index with keys[i] >= key; the key is present by construction
    while (lo < hi) { const unsigned long long mid = (lo + hi) >> 1; if (__ldg(&keys[mid]) < key) lo = mid + 1; else hi = mid; }
    return (unsigned int)lo;
}

__global__ void __launch_bounds__(MESH_THREADS)
mesh_triangle_kernel(const MeshParams p, const unsigned long long* toff, const unsigned long long* keys, unsigned long long n_verts, uint32_t* tris,
                     unsigned long long* cells)
{
    typedef cub::BlockScan<int, MESH_THREADS> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const long long tile = (long long)blockIdx.x * MESH_TILE;
    unsigned long long base = toff[blockIdx.x];
    for (int it = 0; it < MESH_ITEMS; ++it) {
        const long long idx = tile + it * MESH_THREADS + threadIdx.x;
        Voxel v; v.mc_case = -1;
        if (idx < p.total) v = classify(p, idx);
        const int nt = tri_count(v);
        int off, agg;
        Scan(tmp).ExclusiveSum(nt, off, agg);
        uint32_t* o = tris + 3 * (base + (unsigned long long)off);
        if (cells) for (int k = 0; k < nt; ++k) cells[base + (unsigned long long)off + k] = (unsigned long long)idx;
        for (int k = 0; k < 3 * nt; ++k) {
            const int e = kt_mc_tris[v.mc_case][k];
            const int a = e >> 2, j = e & 3;
            // the edge's owner: the cell's lower corner + the edge's offsets on the two other axes (kt_mc_table.h)
            const int ox = a == 0 ? 0 : (j & 1), oy = a == 1 ? 0 : (a == 0 ? (j & 1) : (j >> 1)), oz = a == 2 ? 0 : (j >> 1);
            const long long owner = idx + ox + (long long)p.ex * (oy + (long long)p.ey * oz);
            o[k] = find_vertex(keys, n_verts, 3ull * (unsigned long long)owner + (unsigned long long)a);
        }
        base += (unsigned long long)agg;
        __syncthreads();
    }
}

// the global form of n local keys (see mesh_key_global): edges = vertex keys (3 * owner + axis), else triangle cells (owner)
__global__ void __launch_bounds__(MESH_THREADS)
mesh_global_keys_kernel(const MeshKeyFrame f, const unsigned long long* keys, unsigned long long n, bool edges, int4* out)
{
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = keys[i];
        int g[4];
        mesh_key_global(f, edges ? k / 3 : k, edges ? (int)(k % 3) : 0, g);
        out[i] = make_int4(g[0], g[1], g[2], g[3]);
    }
}

MeshParams make_params(const MeshArgs& a)
{
    MeshParams p;
    p.tsdf = a.tsdf; p.color = (const uchar4*)a.color; p.V = a.vol; p.wrap = wrap_mod3(a.wrap, a.vol); p.real_wrap = a.real_wrap;
    p.cell = make_float3(a.volume_size.x / a.vol, a.volume_size.y / a.vol, a.volume_size.z / a.vol);
    p.inv_cell = make_float3(1.f / p.cell.x, 1.f / p.cell.y, 1.f / p.cell.z);
    p.cull = a.weight_cull;
    p.minX = a.minX; p.maxX = a.maxX; p.minY = a.minY; p.maxY = a.maxY; p.minZ = a.minZ; p.maxZ = a.maxZ;
    p.ex = std::min(a.maxX + 1, a.vol) - a.minX; p.ey = std::min(a.maxY + 1, a.vol) - a.minY;
    const int ez = std::min(a.maxZ + 1, a.vol) - a.minZ;
    p.total = (a.maxX > a.minX && a.maxY > a.minY && a.maxZ > a.minZ) ? (long long)p.ex * p.ey * ez : 0;
    return p;
}

size_t with_slack(size_t n) { return n + n / 4 + 256; }      // capacity of a grown workspace buffer

} // namespace

int mesh_count(const MeshArgs& a, MeshWorkspace* ws, size_t* n_verts, size_t* n_tris, cudaStream_t s)
{
    *n_verts = 0; *n_tris = 0;
    const MeshParams p = make_params(a);
    if (p.total == 0) return 0;
    const long long nb = (p.total + MESH_TILE - 1) / MESH_TILE;
    if (nb > 0x7fffffffLL) { set_error("mesh: box too large"); return KT_ERR_INVALID; }
    const size_t n = (size_t)4 * (nb + 1);
    int r = ws->counts.grow(n, with_slack(n), "mesh tile counts"); if (r) return r;
    if (!ws->totals_host && (r = ws->fixed.pinned(&ws->totals_host, 2, "mesh totals"))) return r;
    unsigned long long* vc = ws->counts.get(); unsigned long long* tc = vc + (nb + 1);
    unsigned long long* vo = tc + (nb + 1); unsigned long long* to = vo + (nb + 1);
    mesh_count_kernel<<<(unsigned int)nb, MESH_THREADS, 0, s>>>(p, vc, tc);
    KT_LAUNCH_CHECK();
    size_t need = 0;
    KT_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, need, vc, vo, (int)(nb + 1), s));
    r = ws->tmp.grow(need, with_slack(need), "mesh scan storage"); if (r) return r;
    size_t have = ws->tmp.capacity();
    KT_CUDA(cub::DeviceScan::ExclusiveSum(ws->tmp.get(), have, vc, vo, (int)(nb + 1), s));
    have = ws->tmp.capacity();
    KT_CUDA(cub::DeviceScan::ExclusiveSum(ws->tmp.get(), have, tc, to, (int)(nb + 1), s));
    KT_CUDA(cudaMemcpyAsync(&ws->totals_host[0], vo + nb, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(&ws->totals_host[1], to + nb, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    *n_verts = (size_t)ws->totals_host[0]; *n_tris = (size_t)ws->totals_host[1];
    return 0;
}

MeshKeyFrame mesh_key_frame(const MeshArgs& a)
{
    MeshKeyFrame f;
    f.min[0] = a.minX; f.min[1] = a.minY; f.min[2] = a.minZ;
    f.ex = std::min(a.maxX + 1, a.vol) - a.minX; f.ey = std::min(a.maxY + 1, a.vol) - a.minY;
    f.real_wrap[0] = a.real_wrap.x; f.real_wrap[1] = a.real_wrap.y; f.real_wrap[2] = a.real_wrap.z;
    return f;
}

int mesh_emit(const MeshArgs& a, MeshWorkspace* ws, size_t n_verts, void* verts, uint32_t* tris, cudaStream_t s, unsigned long long* vkeys,
              unsigned long long* tcells)
{
    const MeshParams p = make_params(a);
    if (p.total == 0 || n_verts == 0) return 0;
    if (n_verts > 0xffffffffull) { set_error("mesh: %zu vertices do not fit 32-bit indices", n_verts); return KT_ERR_CAPACITY; }
    const long long nb = (p.total + MESH_TILE - 1) / MESH_TILE;
    if (!vkeys) { int r = ws->keys.grow(n_verts, with_slack(n_verts), "mesh vertex keys"); if (r) return r; vkeys = ws->keys.get(); }
    const unsigned long long* vo = ws->counts.get() + 2 * (nb + 1); const unsigned long long* to = vo + (nb + 1);
    mesh_vertex_kernel<<<(unsigned int)nb, MESH_THREADS, 0, s>>>(p, vo, (uint4*)verts, vkeys);
    KT_LAUNCH_CHECK();
    mesh_triangle_kernel<<<(unsigned int)nb, MESH_THREADS, 0, s>>>(p, to, vkeys, n_verts, tris, tcells);
    KT_LAUNCH_CHECK();
    return 0;
}

int mesh_global_keys(const MeshArgs& a, const unsigned long long* keys, size_t n, bool edges, int32_t* out, cudaStream_t s)
{
    if (!n) return 0;
    const size_t b = (n + MESH_THREADS - 1) / MESH_THREADS, cap = (size_t)device_info().sm_count * 16;
    mesh_global_keys_kernel<<<(unsigned int)std::min(b, cap), MESH_THREADS, 0, s>>>(mesh_key_frame(a), keys, n, edges, (int4*)out);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
