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

// What the owner voxel idx contributes (mc_classify, kt_surface.cuh): cells are meshed inside the box and away from the far border
struct Voxel { int x, y, z; unsigned int vflags; int mc_case; };

// the volume as kt_surface.cuh's Field: logical voxels, no cyclic wrap
struct BoxField {
    const MeshParams& p;
    __device__ __forceinline__ bool corner(int x, int y, int z, short& raw) const { return kt::corner(p, x, y, z, raw); }
    __device__ __forceinline__ short raw(int x, int y, int z) const { return __ldg(&p.tsdf[vaddr(p, x, y, z)]); }
    __device__ __forceinline__ uchar4 color(int x, int y, int z) const { return __ldg(&p.color[vaddr(p, x, y, z)]); }
};

__device__ __forceinline__ Voxel classify(const MeshParams& p, long long idx)
{
    Voxel v; owner_xyz(p, idx, v.x, v.y, v.z);
    const McVoxel m = mc_classify(BoxField{p}, v.x, v.y, v.z, [&](int cx, int cy, int cz) {
        return cx >= p.minX && cx < p.maxX && cy >= p.minY && cy < p.maxY && cz >= p.minZ && cz < p.maxZ &&
               cx + 1 < p.V && cy + 1 < p.V && cz + 1 < p.V;
    });
    v.vflags = m.vflags; v.mc_case = m.mc_case;
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

__device__ __forceinline__ void write_vertex(const MeshParams& p, int x, int y, int z, int a, uint4* out)
{
    mc_vertex(BoxField{p}, p.cell, p.inv_cell, p.real_wrap, p.V, x, y, z, a, out);
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
