// kintinuous_b200 -- the map volume: a sparse global TSDF of what the moving volume leaves behind, and marching cubes over it.
//
// No counterpart in the reference (it meshes point slices with PCL's GP3).  The slice meshes (kt_mesh.cu) are cut from the TSDF just
// before their planes are cleared, so where two slices disagree about a shared corner the weld (kt_weld.cu) has nothing left to decide
// with and leaves a gap (DESIGN.md R17).  Here the values themselves are kept:
//   * store: just before a shift clears its storage planes (exactly clear_range's: Q13's round_up16 reach on x and the ZMinus slab of
//     Q12 included), every surface voxel of them creates its 8^3 brick, and every voxel with W != 0 overwrites its value in a brick that
//     exists.  S(v), the latest observation of global voxel v (logical voxel + the real voxel wrap), is then the store where the live
//     volume has W = 0, else the live volume.  Bricks without a surface voxel are never stored: such voxels are no valid corner, and
//     marching cubes treats them as unobserved.
//   * hash: open addressing (linear probing) on 64-bit keys, 21 signed bits per brick axis, z most significant, so that ascending keys
//     are bricks in (z, y, x) order.  Slots and pool entries are taken by atomics, so where a brick lands varies; its content does not.
//   * capacity is all or nothing per clear: mark (insert the new keys) -> roll back (when they do not all fit, every key inserted by
//     this clear is removed again; a no-op launch otherwise) -> write (the values; its first thread commits or restores the count and
//     sets `full`).  Three launches per cleared slab on the tracker stream, no host synchronisation, nothing on frames without a shift.
//   * restore (kt_set_map_volume_restore, off by default): once the clear has run, one more launch gives every voxel of the same planes
//     the stored value of its global voxel under the wrap after the shift, where a stored brick holds it with W != 0.  Keys come from
//     coordinates alone (one lookup per distinct key of a warp), so the volume is only written.  The planes Q13 / Q12 clear beyond those
//     that leave keep their global voxels, so their surface bricks come back in the same frame; free space outside stored bricks does not.
//   * export: the live volume's surface bricks and the store's, sorted and made unique with CUB, are merged into one brick set of S
//     (a live voxel with W != 0 wins) -> marching cubes over the brick set: per brick an 11^3 tile of validity and raw values in shared
//     memory (the brick, one voxel below, two above: classification needs the 3x3x3 neighbourhood, the normal of an edge's far end one
//     more), neighbours found by binary search in the sorted keys -> count, scan, emit with kt_surface.cuh's arithmetic (positions as
//     kt_mesh.cu's with the global voxel as the logical one and real wrap 0) -> vertices sorted by (owner voxel in (z, y, x) order,
//     axis) and triangles stably by cell, indices found by binary search.  No atomic decides the output order.  With no shift this is
//     kt_get_live_mesh's mesh byte for byte: outside the live box S is unobserved, exactly like the volume border.
#include "kt_ops.h"
#include "kt_surface.cuh"
#include "../../include/kintinuous_b200.h"
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>
#define KT_MC_STORAGE static __device__ const
#include "kt_mc_table.h"

namespace kt {

namespace {

const int BRICK_THREADS = 512;                      // one thread per voxel of a brick
const int TILE = 11, TILE_VOX = TILE * TILE * TILE; // brick + 1 below + 2 above per axis
const unsigned long long EMPTY_KEY = ~0ull;
const unsigned int NO_BRICK = 0xffffffffu;
const int STORE_THREADS = 256;

__host__ __device__ __forceinline__ unsigned long long key_of(int bx, int by, int bz)
{
    return ((unsigned long long)(bz + MAPVOL_COORD_BIAS) << 42) | ((unsigned long long)(by + MAPVOL_COORD_BIAS) << 21) |
           (unsigned long long)(bx + MAPVOL_COORD_BIAS);
}
__host__ __device__ __forceinline__ int3 brick_of(unsigned long long k)
{
    return make_int3((int)(k & 0x1FFFFFull) - MAPVOL_COORD_BIAS, (int)((k >> 21) & 0x1FFFFFull) - MAPVOL_COORD_BIAS, (int)(k >> 42) - MAPVOL_COORD_BIAS);
}
__host__ __device__ __forceinline__ bool brick_ok(int b) { return b >= -MAPVOL_COORD_BIAS && b < MAPVOL_COORD_BIAS; }
__device__ __forceinline__ int local_of(int gx, int gy, int gz) { return (gx & 7) + 8 * (gy & 7) + 64 * (gz & 7); }

__device__ __forceinline__ unsigned int slot_of(unsigned long long k, unsigned int mask)
{
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (unsigned int)k & mask;
}

struct StoreView {
    unsigned long long* slot_key; unsigned int* slot_val; unsigned int slots, capacity;
    unsigned long long* brick_key; int16_t* tsdf; uchar4* color; unsigned int* state;
};
StoreView view(const MapVolume* m)
{
    StoreView v;
    v.slot_key = m->slot_key; v.slot_val = m->slot_val; v.slots = m->slots; v.capacity = m->capacity;
    v.brick_key = m->brick_key; v.tsdf = m->tsdf; v.color = (uchar4*)m->color; v.state = m->state;
    return v;
}

__device__ __forceinline__ unsigned int lookup(const unsigned long long* slot_key, const unsigned int* slot_val, unsigned int slots, unsigned long long key)
{
    unsigned int h = slot_of(key, slots - 1);
    for (unsigned int probe = 0; probe < slots; ++probe) {
        const unsigned long long k = slot_key[h];
        if (k == key) return slot_val[h];
        if (k == EMPTY_KEY) return NO_BRICK;
        h = (h + 1) & (slots - 1);
    }
    return NO_BRICK;
}

// The voxels a clear zeroes: storage planes [first, first + planes) mod V along `axis`, every row of them; x fastest where x is not the axis.
struct ClearRegion {
    const int16_t* tsdf; const uchar4* color; int V, axis, first, planes; int3 wrap, wbase; long long total;
};
__device__ __forceinline__ void region_voxel(const ClearRegion& r, long long i, int& sx, int& sy, int& sz)
{
    const int V = r.V;
    if (r.axis == 0) {
        const int k = (int)(i % r.planes); const long long row = i / r.planes;
        sx = r.first + k; if (sx >= V) sx -= V;
        sy = (int)(row % V); sz = (int)(row / V);
    } else {
        sx = (int)(i % V); const long long rest = i / V;
        const int o = (int)(rest % V); int p = r.first + (int)(rest / V); if (p >= V) p -= V;
        sy = r.axis == 1 ? p : o; sz = r.axis == 1 ? o : p;
    }
}
// storage coordinate -> global voxel: logical (s - wrap mod V) mod V, plus the signed wrap
__device__ __forceinline__ int global_of(int s, int wbase, int wrap, int V) { int l = s - wbase; if (l < 0) l += V; return l + wrap; }

// brick key of voxel i of the region when it is observed (surface_only: and a surface voxel), else EMPTY_KEY; *refused (may be null) = 1
// for a brick outside the key range
__device__ __forceinline__ unsigned long long region_key(const ClearRegion& r, long long i, bool surface_only, int& gx, int& gy, int& gz,
                                                         short& raw, uchar4& col, unsigned int* refused)
{
    if (i >= r.total) return EMPTY_KEY;
    int sx, sy, sz; region_voxel(r, i, sx, sy, sz);
    const size_t a = ((size_t)sz * r.V + sy) * r.V + sx;
    col = r.color[a];
    if (col.w == 0) return EMPTY_KEY;
    raw = r.tsdf[a];
    if (surface_only && !surface_voxel(col.w, unpack_tsdf(raw))) return EMPTY_KEY;
    gx = global_of(sx, r.wbase.x, r.wrap.x, r.V); gy = global_of(sy, r.wbase.y, r.wrap.y, r.V); gz = global_of(sz, r.wbase.z, r.wrap.z, r.V);
    const int bx = gx >> 3, by = gy >> 3, bz = gz >> 3;
    if (!brick_ok(bx) || !brick_ok(by) || !brick_ok(bz)) { if (refused) atomicExch(refused, 1u); return EMPTY_KEY; }
    return key_of(bx, by, bz);
}

// 1: insert the brick of every surface voxel (one lane per distinct key of a warp).  state[0] counts the bricks taken, state[2] = 1 when
// a probe found no free slot or a brick is out of range.
__global__ void __launch_bounds__(STORE_THREADS)
mapvol_mark_kernel(const ClearRegion r, const StoreView m)
{
    const unsigned int lane = threadIdx.x & 31;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < r.total; base += (long long)gridDim.x * blockDim.x) {
        int gx, gy, gz; short raw; uchar4 col;
        const unsigned long long key = region_key(r, base + threadIdx.x, true, gx, gy, gz, raw, col, &m.state[2]);
        const unsigned int same = __match_any_sync(0xffffffffu, key);
        if (key == EMPTY_KEY || (unsigned int)(__ffs(same) - 1) != lane) continue;
        unsigned int h = slot_of(key, m.slots - 1);
        bool placed = false;
        for (unsigned int probe = 0; probe < m.slots && !placed; ++probe) {
            const unsigned long long k = *(volatile unsigned long long*)&m.slot_key[h];
            if (k == key) placed = true;
            else if (k == EMPTY_KEY) {
                const unsigned long long prev = atomicCAS(&m.slot_key[h], EMPTY_KEY, key);
                if (prev == EMPTY_KEY) {
                    const unsigned int idx = atomicAdd(&m.state[0], 1u);
                    m.slot_val[h] = idx;
                    if (idx < m.capacity) m.brick_key[idx] = key;
                    placed = true;
                } else if (prev == key) placed = true;
            }
            h = (h + 1) & (m.slots - 1);
        }
        if (!placed) atomicExch(&m.state[2], 1u);
    }
}

// 2: when this clear's bricks do not all fit, remove every key it inserted (pool index >= the committed count).  Keys inserted before
// it never probed past a newer one, so the table is exactly what it was.
__global__ void __launch_bounds__(STORE_THREADS)
mapvol_rollback_kernel(const StoreView m)
{
    const unsigned int count = m.state[0], committed = m.state[1];
    if (count <= m.capacity && m.state[2] == 0) return;
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s < m.slots; s += gridDim.x * blockDim.x)
        if (m.slot_key[s] != EMPTY_KEY && m.slot_val[s] >= committed) m.slot_key[s] = EMPTY_KEY;
}

// 3: every observed voxel of the region overwrites its value in a brick that exists; the first thread commits the count (or restores
// it and sets full)
__global__ void __launch_bounds__(STORE_THREADS)
mapvol_write_kernel(const ClearRegion r, const StoreView m)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (m.state[0] > m.capacity || m.state[2]) { m.state[0] = m.state[1]; m.state[3] = 1u; m.state[2] = 0u; }
        else m.state[1] = m.state[0];
    }
    const unsigned int lane = threadIdx.x & 31;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < r.total; base += (long long)gridDim.x * blockDim.x) {
        int gx = 0, gy = 0, gz = 0; short raw = 0; uchar4 col;
        const unsigned long long key = region_key(r, base + threadIdx.x, false, gx, gy, gz, raw, col, nullptr);
        const unsigned int same = __match_any_sync(0xffffffffu, key);
        const int leader = __ffs(same) - 1;
        unsigned int b = NO_BRICK;
        if (key != EMPTY_KEY && (int)lane == leader) b = lookup(m.slot_key, m.slot_val, m.slots, key);
        b = __shfl_sync(0xffffffffu, b, leader);
        if (key == EMPTY_KEY || b == NO_BRICK) continue;
        const size_t at = (size_t)b * MAPVOL_BRICK_VOXELS + local_of(gx, gy, gz);
        m.tsdf[at] = raw; m.color[at] = col;
    }
}

// restore, after the clear: every voxel of the region (r.wrap = the wrap after the shift) whose global voxel has a stored value with
// W != 0 takes that value.  Keys come from coordinates alone, so the volume is only written; no atomics.
__global__ void __launch_bounds__(STORE_THREADS)
mapvol_restore_kernel(const ClearRegion r, const StoreView m, int16_t* tsdf, uchar4* color)
{
    const unsigned int lane = threadIdx.x & 31;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < r.total; base += (long long)gridDim.x * blockDim.x) {
        const long long i = base + threadIdx.x;
        int sx = 0, sy = 0, sz = 0, gx = 0, gy = 0, gz = 0;
        unsigned long long key = EMPTY_KEY;
        if (i < r.total) {
            region_voxel(r, i, sx, sy, sz);
            gx = global_of(sx, r.wbase.x, r.wrap.x, r.V); gy = global_of(sy, r.wbase.y, r.wrap.y, r.V); gz = global_of(sz, r.wbase.z, r.wrap.z, r.V);
            if (brick_ok(gx >> 3) && brick_ok(gy >> 3) && brick_ok(gz >> 3)) key = key_of(gx >> 3, gy >> 3, gz >> 3);
        }
        const unsigned int same = __match_any_sync(0xffffffffu, key);
        const int leader = __ffs(same) - 1;
        unsigned int b = NO_BRICK;
        if (key != EMPTY_KEY && (int)lane == leader) b = lookup(m.slot_key, m.slot_val, m.slots, key);
        b = __shfl_sync(0xffffffffu, b, leader);
        if (b == NO_BRICK) continue;
        const size_t at = (size_t)b * MAPVOL_BRICK_VOXELS + local_of(gx, gy, gz);
        const uchar4 col = m.color[at];
        if (col.w == 0) continue;
        const size_t a = ((size_t)sz * r.V + sy) * r.V + sx;
        tsdf[a] = m.tsdf[at]; color[a] = col;
    }
}

// ---- export: the merged brick set ----
struct LiveBox { const int16_t* tsdf; const uchar4* color; int V; int3 wrap, wbase; int3 b0; int nbx, nby; };

__device__ __forceinline__ bool live_voxel(const LiveBox& L, int gx, int gy, int gz, size_t& a)
{
    const int lx = gx - L.wrap.x, ly = gy - L.wrap.y, lz = gz - L.wrap.z;
    if ((unsigned)lx >= (unsigned)L.V || (unsigned)ly >= (unsigned)L.V || (unsigned)lz >= (unsigned)L.V) return false;
    int sx = lx + L.wbase.x; if (sx >= L.V) sx -= L.V;
    int sy = ly + L.wbase.y; if (sy >= L.V) sy -= L.V;
    int sz = lz + L.wbase.z; if (sz >= L.V) sz -= L.V;
    a = ((size_t)sz * L.V + sy) * L.V + sx;
    return true;
}

// per brick overlapping the live box: its key, and whether it holds a surface voxel of the live volume
__global__ void __launch_bounds__(BRICK_THREADS)
live_bricks_kernel(const LiveBox L, unsigned long long* keys, unsigned char* flags)
{
    const int b = blockIdx.x;
    const int bx = L.b0.x + b % L.nbx, by = L.b0.y + (b / L.nbx) % L.nby, bz = L.b0.z + b / (L.nbx * L.nby);
    const int t = threadIdx.x;
    const int gx = 8 * bx + (t & 7), gy = 8 * by + ((t >> 3) & 7), gz = 8 * bz + (t >> 6);
    size_t a; bool s = false;
    if (live_voxel(L, gx, gy, gz, a)) { const int W = L.color[a].w; s = surface_voxel(W, unpack_tsdf(L.tsdf[a])); }
    s = __syncthreads_or(s);
    if (t == 0) { keys[b] = key_of(bx, by, bz); flags[b] = s ? 1 : 0; }
}

// S over every brick of the sorted unique set: the live voxel where it is observed, else the store's value, else unobserved
__global__ void __launch_bounds__(BRICK_THREADS)
merge_bricks_kernel(const LiveBox L, const StoreView m, bool with_store, const unsigned long long* keys, int16_t* tsdf, uchar4* color)
{
    __shared__ unsigned int sb;
    const unsigned long long key = keys[blockIdx.x];
    if (threadIdx.x == 0) sb = with_store ? lookup(m.slot_key, m.slot_val, m.slots, key) : NO_BRICK;
    __syncthreads();
    const int3 b = brick_of(key);
    const int t = threadIdx.x;
    const int gx = 8 * b.x + (t & 7), gy = 8 * b.y + ((t >> 3) & 7), gz = 8 * b.z + (t >> 6);
    short raw = 0; uchar4 c = make_uchar4(0, 0, 0, 0);
    size_t a;
    if (live_voxel(L, gx, gy, gz, a) && L.color[a].w != 0) { raw = L.tsdf[a]; c = L.color[a]; }
    else if (sb != NO_BRICK) { const size_t at = (size_t)sb * MAPVOL_BRICK_VOXELS + t; raw = m.tsdf[at]; c = m.color[at]; }
    const size_t o = (size_t)blockIdx.x * MAPVOL_BRICK_VOXELS + t;
    tsdf[o] = raw; color[o] = c;
}

// ---- marching cubes over a sorted brick set ----
struct BrickGrid {
    const unsigned long long* keys; const int16_t* tsdf; const uchar4* color; unsigned int n; int cull;
    float3 cell, inv_cell; int V;
    int min[3]; unsigned long long ex, exy;            // dense global voxel index relative to min, x fastest
};

__device__ __forceinline__ unsigned int find_brick(const unsigned long long* keys, unsigned int n, unsigned long long key)
{
    unsigned int lo = 0, hi = n;
    while (lo < hi) { const unsigned int mid = (lo + hi) >> 1; if (__ldg(&keys[mid]) < key) lo = mid + 1; else hi = mid; }
    return lo < n && __ldg(&keys[lo]) == key ? lo : NO_BRICK;
}

struct Tile { short raw[TILE_VOX]; unsigned char ok[TILE_VOX]; unsigned int nb[27]; };

// one brick's tile: entry (i, j, k) is global voxel 8 * brick - 1 + (i, j, k)
__device__ __forceinline__ void load_tile(const BrickGrid& g, int3 b, Tile& T)
{
    if (threadIdx.x < 27) {
        const int dx = (int)threadIdx.x % 3 - 1, dy = ((int)threadIdx.x / 3) % 3 - 1, dz = (int)threadIdx.x / 9 - 1;
        const int nx = b.x + dx, ny = b.y + dy, nz = b.z + dz;
        T.nb[threadIdx.x] = brick_ok(nx) && brick_ok(ny) && brick_ok(nz) ? find_brick(g.keys, g.n, key_of(nx, ny, nz)) : NO_BRICK;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < TILE_VOX; e += BRICK_THREADS) {
        const int i = e % TILE, j = (e / TILE) % TILE, k = e / (TILE * TILE);
        const int lx = i - 1, ly = j - 1, lz = k - 1;                      // -1 .. 9 relative to the brick
        const int ox = lx < 0 ? 0 : lx < 8 ? 1 : 2, oy = ly < 0 ? 0 : ly < 8 ? 1 : 2, oz = lz < 0 ? 0 : lz < 8 ? 1 : 2;
        const unsigned int nb = T.nb[ox + 3 * oy + 9 * oz];
        short raw = 0; bool ok = false;
        if (nb != NO_BRICK) {
            const size_t at = (size_t)nb * MAPVOL_BRICK_VOXELS + ((lx + 8) & 7) + 8 * ((ly + 8) & 7) + 64 * ((lz + 8) & 7);
            raw = __ldg(&g.tsdf[at]);
            const int W = __ldg(&g.color[at]).w;
            ok = surface_voxel(W, unpack_tsdf(raw)) && W >= g.cull;
        }
        T.raw[e] = raw; T.ok[e] = ok ? 1 : 0;
    }
    __syncthreads();
}

// the tile as kt_surface.cuh's Field, in global voxel coordinates
struct TileField {
    const Tile& T; const BrickGrid& g; int ox, oy, oz;            // global voxel of tile entry (0, 0, 0)
    __device__ __forceinline__ int at(int x, int y, int z) const { return (x - ox) + TILE * ((y - oy) + TILE * (z - oz)); }
    __device__ __forceinline__ bool corner(int x, int y, int z, short& raw) const
    {
        const int e = at(x, y, z);
        if (!T.ok[e]) return false;
        raw = T.raw[e]; return true;
    }
    __device__ __forceinline__ short raw(int x, int y, int z) const { return T.raw[at(x, y, z)]; }
    __device__ __forceinline__ uchar4 color(int x, int y, int z) const
    {
        const int lx = x - ox - 1, ly = y - oy - 1, lz = z - oz - 1;
        const int bx = lx < 0 ? 0 : lx < 8 ? 1 : 2, by = ly < 0 ? 0 : ly < 8 ? 1 : 2, bz = lz < 0 ? 0 : lz < 8 ? 1 : 2;
        const size_t a = (size_t)T.nb[bx + 3 * by + 9 * bz] * MAPVOL_BRICK_VOXELS + ((lx + 8) & 7) + 8 * ((ly + 8) & 7) + 64 * ((lz + 8) & 7);
        return __ldg(&g.color[a]);
    }
};

struct AnyCell { __device__ __forceinline__ bool operator()(int, int, int) const { return true; } };

__device__ __forceinline__ unsigned long long dense(const BrickGrid& g, int x, int y, int z)
{
    return (unsigned long long)(x - g.min[0]) + (unsigned long long)(y - g.min[1]) * g.ex + (unsigned long long)(z - g.min[2]) * g.exy;
}

// per-brick vertex / triangle counts; entry n (one past the last) gets 0 so that the exclusive scans end in the totals
__global__ void __launch_bounds__(BRICK_THREADS)
brick_count_kernel(const BrickGrid g, unsigned long long* vcount, unsigned long long* tcount)
{
    __shared__ Tile T;
    typedef cub::BlockReduce<int, BRICK_THREADS> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const int3 b = brick_of(g.keys[blockIdx.x]);
    load_tile(g, b, T);
    const TileField f{T, g, 8 * b.x - 1, 8 * b.y - 1, 8 * b.z - 1};
    const int t = threadIdx.x;
    const McVoxel v = mc_classify(f, 8 * b.x + (t & 7), 8 * b.y + ((t >> 3) & 7), 8 * b.z + (t >> 6), AnyCell());
    const int nv = __popc(v.vflags), nt = v.mc_case < 0 ? 0 : kt_mc_tri_count[v.mc_case];
    const int sv = Reduce(tmp).Sum(nv);
    __syncthreads();
    const int st = Reduce(tmp).Sum(nt);
    if (t == 0) {
        vcount[blockIdx.x] = (unsigned long long)sv; tcount[blockIdx.x] = (unsigned long long)st;
        if (blockIdx.x == 0) { vcount[gridDim.x] = 0; tcount[gridDim.x] = 0; }
    }
}

// vertices (in brick order) with their keys 3 * dense(owner) + axis; triangles with their cell key dense(cell) and the keys of their 3 edges
__global__ void __launch_bounds__(BRICK_THREADS)
brick_emit_kernel(const BrickGrid g, const unsigned long long* voff, const unsigned long long* toff, uint4* verts, unsigned long long* vkeys,
                  unsigned int* vidx, unsigned long long* tcell, unsigned int* tidx, unsigned long long* tedge)
{
    __shared__ Tile T;
    typedef cub::BlockScan<int, BRICK_THREADS> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const int3 b = brick_of(g.keys[blockIdx.x]);
    load_tile(g, b, T);
    const TileField f{T, g, 8 * b.x - 1, 8 * b.y - 1, 8 * b.z - 1};
    const int t = threadIdx.x;
    const int x = 8 * b.x + (t & 7), y = 8 * b.y + ((t >> 3) & 7), z = 8 * b.z + (t >> 6);
    const McVoxel v = mc_classify(f, x, y, z, AnyCell());
    const int nt = v.mc_case < 0 ? 0 : kt_mc_tri_count[v.mc_case];
    int off, agg;
    Scan(tmp).ExclusiveSum(__popc(v.vflags), off, agg);
    unsigned long long slot = voff[blockIdx.x] + (unsigned long long)off;
    const unsigned long long owner = dense(g, x, y, z);
    for (int a = 0; a < 3; ++a)
        if (v.vflags & (1u << a)) {
            mc_vertex(f, g.cell, g.inv_cell, make_int3(0, 0, 0), g.V, x, y, z, a, verts + 2 * slot);
            vkeys[slot] = 3ull * owner + (unsigned long long)a; vidx[slot] = (unsigned int)slot;
            ++slot;
        }
    __syncthreads();
    Scan(tmp).ExclusiveSum(nt, off, agg);
    const unsigned long long tb = toff[blockIdx.x] + (unsigned long long)off;
    for (int k = 0; k < nt; ++k) {
        tcell[tb + k] = owner; tidx[tb + k] = (unsigned int)(tb + k);
        for (int c = 0; c < 3; ++c) {
            const int e = kt_mc_tris[v.mc_case][3 * k + c];
            const int a = e >> 2, j = e & 3;
            // the edge's owner: the cell's lower corner + the edge's offsets on the two other axes (kt_mc_table.h)
            const int ox = a == 0 ? 0 : (j & 1), oy = a == 1 ? 0 : (a == 0 ? (j & 1) : (j >> 1)), oz = a == 2 ? 0 : (j >> 1);
            tedge[3 * (tb + k) + c] = 3ull * dense(g, x + ox, y + oy, z + oz) + (unsigned long long)a;
        }
    }
}

// keys strictly ascending and inside the key range; bounds[0..2] = min, [3..5] = max brick coordinate, [6] = bad keys
__global__ void __launch_bounds__(256)
brick_bounds_kernel(const unsigned long long* keys, unsigned int n, int* bounds)
{
    int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {INT_MIN, INT_MIN, INT_MIN}, bad = 0;
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long k = keys[i];
        if ((k >> 63) || (i + 1 < n && keys[i + 1] <= k)) ++bad;
        const int3 b = brick_of(k);
        mn[0] = min(mn[0], b.x); mn[1] = min(mn[1], b.y); mn[2] = min(mn[2], b.z);
        mx[0] = max(mx[0], b.x); mx[1] = max(mx[1], b.y); mx[2] = max(mx[2], b.z);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o)); mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o)); }
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { atomicMin(&bounds[a], mn[a]); atomicMax(&bounds[3 + a], mx[a]); }
        if (bad) atomicAdd(&bounds[6], bad);
    }
}

__global__ void __launch_bounds__(256)
gather_verts_kernel(const uint4* verts, const unsigned int* order, unsigned int n, uint4* out)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const unsigned int v = order[i]; out[2 * i] = verts[2 * v]; out[2 * i + 1] = verts[2 * v + 1]; }
}

__global__ void __launch_bounds__(256)
write_tris_kernel(const unsigned int* order, unsigned int n, const unsigned long long* tedge, const unsigned long long* vkeys, unsigned int nv, uint32_t* out)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned int t = order[i];
    for (int c = 0; c < 3; ++c) {
        const unsigned long long key = tedge[3 * (size_t)t + c];
        unsigned int lo = 0, hi = nv;                  // first index with vkeys[i] >= key; present by construction
        while (lo < hi) { const unsigned int mid = (lo + hi) >> 1; if (__ldg(&vkeys[mid]) < key) lo = mid + 1; else hi = mid; }
        out[3 * (size_t)i + c] = lo;
    }
}

__global__ void __launch_bounds__(256)
gather_store_kernel(const unsigned int* order, unsigned int n, const StoreView m, int16_t* tsdf, uchar4* color)
{
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned long long)n * MAPVOL_BRICK_VOXELS) return;
    const size_t from = (size_t)order[i / MAPVOL_BRICK_VOXELS] * MAPVOL_BRICK_VOXELS + i % MAPVOL_BRICK_VOXELS;
    tsdf[i] = m.tsdf[from]; color[i] = m.color[from];
}

int key_bits(unsigned long long kmax) { int b = 1; while (b < 64 && (kmax >> b) != 0) ++b; return b; }
unsigned int blocks_for(size_t n, int threads = 256) { return (unsigned int)((n + threads - 1) / threads); }
unsigned int grid_for(size_t n)
{
    const size_t b = (n + STORE_THREADS - 1) / STORE_THREADS, cap = (size_t)device_info().sm_count * 16;
    return (unsigned int)std::max<size_t>(1, std::min(b, cap));
}

} // namespace

int mapvol_init(MapVolume* m, size_t max_bricks, cudaStream_t s)
{
    const char* who = "kt_set_map_volume";
    if (max_bricks == 0 || max_bricks > 0x40000000ull) { set_error("%s: max_bricks %zu outside 1 .. 2^30", who, max_bricks); return KT_ERR_INVALID; }
    unsigned int slots = 1024;
    while (slots < 2 * max_bricks) slots <<= 1;
    m->capacity = (unsigned int)max_bricks; m->slots = slots;
    if (m->mem.device(&m->slot_key, slots, who) || m->mem.device(&m->slot_val, slots, who) || m->mem.device(&m->brick_key, max_bricks, who) ||
        m->mem.device(&m->tsdf, max_bricks * MAPVOL_BRICK_VOXELS, who) || m->mem.device(&m->color, max_bricks * MAPVOL_BRICK_VOXELS * 4, who) ||
        m->mem.device(&m->state, 4, who) || m->mem.pinned(&m->state_host, 4, who)) return KT_ERR_CUDA;
    return mapvol_empty(m, s);
}

int mapvol_empty(MapVolume* m, cudaStream_t s)
{
    KT_CUDA(cudaMemsetAsync(m->slot_key, 0xff, (size_t)m->slots * sizeof(unsigned long long), s));
    KT_CUDA(cudaMemsetAsync(m->tsdf, 0, (size_t)m->capacity * MAPVOL_BRICK_VOXELS * 2, s));
    KT_CUDA(cudaMemsetAsync(m->color, 0, (size_t)m->capacity * MAPVOL_BRICK_VOXELS * 4, s));
    KT_CUDA(cudaMemsetAsync(m->state, 0, 4 * sizeof(unsigned int), s));
    return 0;
}

int mapvol_store(MapVolume* m, const int16_t* tsdf, const uint8_t* color, int vol, const int* wrap, int axis, int first, int planes, cudaStream_t s)
{
    if (planes <= 0) return 0;
    ClearRegion r;
    r.tsdf = tsdf; r.color = (const uchar4*)color; r.V = vol; r.axis = axis; r.first = first; r.planes = planes;
    r.wrap = make_int3(wrap[0], wrap[1], wrap[2]); r.wbase = wrap_mod3(r.wrap, vol);
    r.total = (long long)planes * vol * vol;
    const StoreView v = view(m);
    const unsigned int grid = grid_for((size_t)r.total);
    mapvol_mark_kernel<<<grid, STORE_THREADS, 0, s>>>(r, v);
    KT_LAUNCH_CHECK();
    mapvol_rollback_kernel<<<grid_for(m->slots), STORE_THREADS, 0, s>>>(v);
    KT_LAUNCH_CHECK();
    mapvol_write_kernel<<<grid, STORE_THREADS, 0, s>>>(r, v);
    KT_LAUNCH_CHECK();
    return 0;
}

int mapvol_restore(MapVolume* m, int16_t* tsdf, uint8_t* color, int vol, const int* wrap_after, int axis, int first, int planes, cudaStream_t s)
{
    if (planes <= 0) return 0;
    ClearRegion r;
    r.tsdf = nullptr; r.color = nullptr; r.V = vol; r.axis = axis; r.first = first; r.planes = planes;
    r.wrap = make_int3(wrap_after[0], wrap_after[1], wrap_after[2]); r.wbase = wrap_mod3(r.wrap, vol);
    r.total = (long long)planes * vol * vol;
    mapvol_restore_kernel<<<grid_for((size_t)r.total), STORE_THREADS, 0, s>>>(r, view(m), tsdf, (uchar4*)color);
    KT_LAUNCH_CHECK();
    return 0;
}

int mapvol_info(MapVolume* m, size_t* bricks, int* full, cudaStream_t s)
{
    KT_CUDA(cudaMemcpyAsync(m->state_host, m->state, 4 * sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    *bricks = m->state_host[1]; *full = m->state_host[3] ? 1 : 0;
    return 0;
}

int mapvol_bricks(MapVolume* m, unsigned long long* keys, int16_t* tsdf, uint8_t* color, size_t max, size_t* n, cudaStream_t s)
{
    const char* who = "kt_get_map_volume_bricks";
    size_t nb = 0; int full = 0;
    int r = mapvol_info(m, &nb, &full, s); if (r) return r;
    *n = nb;
    if (!nb || (!keys && !tsdf && !color)) return 0;
    if (nb > max) { set_error("%s: %zu bricks exceed the capacity %zu", who, nb, max); return KT_ERR_CAPACITY; }
    Allocations mem(s);
    unsigned long long *k1; unsigned int *i0, *i1; int16_t* t; uint8_t* c; unsigned char* tmp;
    if (mem.device(&k1, nb, who) || mem.device(&i0, nb, who) || mem.device(&i1, nb, who) || mem.device(&t, nb * MAPVOL_BRICK_VOXELS, who) ||
        mem.device(&c, nb * MAPVOL_BRICK_VOXELS * 4, who)) return KT_ERR_CUDA;
    std::vector<unsigned int> iota(nb);
    for (size_t i = 0; i < nb; ++i) iota[i] = (unsigned int)i;
    KT_CUDA(cudaMemcpyAsync(i0, iota.data(), nb * sizeof(unsigned int), cudaMemcpyHostToDevice, s));
    size_t need = 0;
    KT_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, need, m->brick_key, k1, i0, i1, (int)nb, 0, 63, s));
    if (mem.device(&tmp, need, who)) return KT_ERR_CUDA;
    KT_CUDA(cub::DeviceRadixSort::SortPairs(tmp, need, m->brick_key, k1, i0, i1, (int)nb, 0, 63, s));
    gather_store_kernel<<<blocks_for(nb * MAPVOL_BRICK_VOXELS), 256, 0, s>>>(i1, (unsigned int)nb, view(m), t, (uchar4*)c);
    KT_LAUNCH_CHECK();
    if (keys) KT_CUDA(cudaMemcpyAsync(keys, k1, nb * 8, cudaMemcpyDeviceToHost, s));
    if (tsdf) KT_CUDA(cudaMemcpyAsync(tsdf, t, nb * MAPVOL_BRICK_VOXELS * 2, cudaMemcpyDeviceToHost, s));
    if (color) KT_CUDA(cudaMemcpyAsync(color, c, nb * MAPVOL_BRICK_VOXELS * 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    return 0;
}

int mesh_bricks(const BrickSet& set, const float3& volume_size, int vol, int weight_cull, const MeshOutput& out, size_t* n_verts, size_t* n_tris,
                float* ms, cudaStream_t s)
{
    const char* who = "mesh_bricks";
    *n_verts = 0; *n_tris = 0;
    if (set.n == 0) { void* v = nullptr; uint32_t* t = nullptr; const int o = out(0, 0, &v, &t); return o < 0 ? o : 0; }
    if (set.n > 0x7fffffffull) { set_error("%s: %zu bricks, at most 2^31 - 1", who, set.n); return KT_ERR_INVALID; }
    const unsigned int N = (unsigned int)set.n;
    Allocations mem(s);
    cudaEvent_t ev[4];
    for (int e = 0; e < 4; ++e) if (mem.event(&ev[e], cudaEventDefault, who)) return KT_ERR_CUDA;
    int* bounds; unsigned long long* counts;
    if (mem.device(&bounds, 8, who) || mem.device(&counts, 4 * ((size_t)N + 1), who)) return KT_ERR_CUDA;
    int host[8] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN, 0, 0};
    KT_CUDA(cudaEventRecord(ev[0], s));
    KT_CUDA(cudaMemcpyAsync(bounds, host, sizeof(host), cudaMemcpyHostToDevice, s));
    brick_bounds_kernel<<<grid_for(N), 256, 0, s>>>(set.keys, N, bounds);
    KT_LAUNCH_CHECK();
    KT_CUDA(cudaMemcpyAsync(host, bounds, sizeof(host), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    if (host[6]) { set_error("%s: %d brick keys are not strictly ascending or outside the 21-bit range", who, host[6]); return KT_ERR_INVALID; }
    BrickGrid g;
    g.keys = set.keys; g.tsdf = set.tsdf; g.color = (const uchar4*)set.color; g.n = N; g.cull = weight_cull; g.V = vol;
    g.cell = make_float3(volume_size.x / vol, volume_size.y / vol, volume_size.z / vol);
    g.inv_cell = make_float3(1.f / g.cell.x, 1.f / g.cell.y, 1.f / g.cell.z);
    unsigned long long ext[3];
    for (int a = 0; a < 3; ++a) { g.min[a] = 8 * host[a]; ext[a] = 8ull * (unsigned long long)((long long)host[3 + a] - host[a] + 1) + 1; }
    const unsigned long long LIM = 1ull << 62;
    if (ext[1] > LIM / ext[0] || ext[2] > LIM / (ext[0] * ext[1]) || ext[0] * ext[1] * ext[2] > LIM / 3) {
        set_error("%s: the bricks span %llu x %llu x %llu voxels, beyond 2^62 edge keys", who, ext[0], ext[1], ext[2]); return KT_ERR_INVALID;
    }
    g.ex = ext[0]; g.exy = ext[0] * ext[1];
    const int ebits = key_bits(3 * g.exy * ext[2] - 1);

    unsigned long long *vc = counts, *tc = vc + (N + 1), *vo = tc + (N + 1), *to = vo + (N + 1);
    brick_count_kernel<<<N, BRICK_THREADS, 0, s>>>(g, vc, tc);
    KT_LAUNCH_CHECK();
    unsigned char* tmp; size_t scan = 0;
    KT_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan, vc, vo, (int)(N + 1), s));
    if (mem.device(&tmp, scan, who)) return KT_ERR_CUDA;
    size_t have = scan;
    KT_CUDA(cub::DeviceScan::ExclusiveSum(tmp, have, vc, vo, (int)(N + 1), s));
    have = scan;
    KT_CUDA(cub::DeviceScan::ExclusiveSum(tmp, have, tc, to, (int)(N + 1), s));
    unsigned long long tot[2];
    KT_CUDA(cudaMemcpyAsync(&tot[0], vo + N, 8, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(&tot[1], to + N, 8, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const size_t nv = (size_t)tot[0], nt = (size_t)tot[1];
    *n_verts = nv; *n_tris = nt;
    if (nv > 0x7fffffffull || nt > 0x7fffffffull) { set_error("%s: %zu vertices / %zu triangles, at most 2^31 - 1 each", who, nv, nt); return KT_ERR_CAPACITY; }
    void* verts_out = nullptr; uint32_t* tris_out = nullptr;
    const int o = out(nv, nt, &verts_out, &tris_out);
    if (o < 0) return o;
    KT_CUDA(cudaEventRecord(ev[1], s));
    if (o == 0 && nv) {
        uint4* verts; unsigned long long *vk0, *vk1, *tc0, *tc1, *tedge; unsigned int *vi0, *vi1, *ti0, *ti1; unsigned char* stmp;
        const size_t ntt = std::max<size_t>(nt, 1);
        if (mem.device(&verts, 2 * nv, who) || mem.device(&vk0, nv, who) || mem.device(&vk1, nv, who) || mem.device(&vi0, nv, who) ||
            mem.device(&vi1, nv, who) || mem.device(&tc0, ntt, who) || mem.device(&tc1, ntt, who) || mem.device(&ti0, ntt, who) ||
            mem.device(&ti1, ntt, who) || mem.device(&tedge, 3 * ntt, who)) return KT_ERR_CUDA;
        brick_emit_kernel<<<N, BRICK_THREADS, 0, s>>>(g, vo, to, verts, vk0, vi0, tc0, ti0, tedge);
        KT_LAUNCH_CHECK();
        KT_CUDA(cudaEventRecord(ev[2], s));
        cub::DoubleBuffer<unsigned long long> vkb(vk0, vk1), tkb(tc0, tc1); cub::DoubleBuffer<unsigned int> vib(vi0, vi1), tib(ti0, ti1);
        size_t sv = 0, st = 0;
        KT_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sv, vkb, vib, (int)nv, 0, ebits, s));
        KT_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, st, tkb, tib, (int)ntt, 0, ebits, s));
        const size_t sbytes = std::max(sv, st);
        if (mem.device(&stmp, sbytes, who)) return KT_ERR_CUDA;
        have = sbytes;
        KT_CUDA(cub::DeviceRadixSort::SortPairs(stmp, have, vkb, vib, (int)nv, 0, ebits, s));
        if (nt) { have = sbytes; KT_CUDA(cub::DeviceRadixSort::SortPairs(stmp, have, tkb, tib, (int)nt, 0, ebits, s)); }
        gather_verts_kernel<<<blocks_for(nv), 256, 0, s>>>(verts, vib.Current(), (unsigned int)nv, (uint4*)verts_out);
        KT_LAUNCH_CHECK();
        if (nt) {
            write_tris_kernel<<<blocks_for(nt), 256, 0, s>>>(tib.Current(), (unsigned int)nt, tedge, vkb.Current(), (unsigned int)nv, tris_out);
            KT_LAUNCH_CHECK();
        }
    } else KT_CUDA(cudaEventRecord(ev[2], s));
    KT_CUDA(cudaEventRecord(ev[3], s));
    KT_CUDA(cudaStreamSynchronize(s));
    if (ms) {
        float a = 0, b = 0, c = 0;
        KT_CUDA(cudaEventElapsedTime(&a, ev[0], ev[2]));       // bounds, count, scan, emit
        KT_CUDA(cudaEventElapsedTime(&b, ev[2], ev[3]));       // sorts and index search
        KT_CUDA(cudaEventElapsedTime(&c, ev[0], ev[3]));
        ms[0] = a; ms[1] = b; ms[2] = c;
    }
    return 0;
}

int mapvol_mesh(const MapVolume* m, const int16_t* tsdf, const uint8_t* color, int vol, const int* wrap, const float3& volume_size, int weight_cull,
                const MeshOutput& out, size_t* n_verts, size_t* n_tris, kt_global_mesh_report* rep, cudaStream_t s)
{
    const char* who = "kt_get_global_mesh";
    *n_verts = 0; *n_tris = 0;
    LiveBox L;
    L.tsdf = tsdf; L.color = (const uchar4*)color; L.V = vol; L.wrap = make_int3(wrap[0], wrap[1], wrap[2]); L.wbase = wrap_mod3(L.wrap, vol);
    const int lo[3] = {wrap[0] >> 3, wrap[1] >> 3, wrap[2] >> 3}, hi[3] = {(wrap[0] + vol - 1) >> 3, (wrap[1] + vol - 1) >> 3, (wrap[2] + vol - 1) >> 3};
    for (int a = 0; a < 3; ++a)
        if (!brick_ok(lo[a]) || !brick_ok(hi[a])) { set_error("%s: the volume's wrap %d lies outside the 21-bit brick range", who, wrap[a]); return KT_ERR_INVALID; }
    L.b0 = make_int3(lo[0], lo[1], lo[2]); L.nbx = hi[0] - lo[0] + 1; L.nby = hi[1] - lo[1] + 1;
    const size_t n_live_box = (size_t)L.nbx * L.nby * (hi[2] - lo[2] + 1);
    Allocations mem(s);
    cudaEvent_t ev[2];
    for (int e = 0; e < 2; ++e) if (mem.event(&ev[e], cudaEventDefault, who)) return KT_ERR_CUDA;
    size_t n_store = 0; int full = 0;
    const StoreView v = view(m);
    int r = mapvol_info(const_cast<MapVolume*>(m), &n_store, &full, s); if (r) return r;
    KT_CUDA(cudaEventRecord(ev[0], s));
    // candidates: the store's keys, then the live box's surface bricks; sorted, unique
    const size_t ncand = n_store + n_live_box;
    unsigned long long *cand, *lkeys, *sorted, *uniq; unsigned char* lflags; int* nsel; unsigned char* tmp;
    if (mem.device(&cand, ncand, who) || mem.device(&lkeys, n_live_box, who) || mem.device(&lflags, n_live_box, who) ||
        mem.device(&sorted, ncand, who) || mem.device(&uniq, ncand, who) || mem.device(&nsel, 2, who)) return KT_ERR_CUDA;
    live_bricks_kernel<<<(unsigned int)n_live_box, BRICK_THREADS, 0, s>>>(L, lkeys, lflags);
    KT_LAUNCH_CHECK();
    if (n_store) KT_CUDA(cudaMemcpyAsync(cand, m->brick_key, n_store * 8, cudaMemcpyDeviceToDevice, s));
    size_t b_sel = 0, b_sort = 0, b_uniq = 0;
    KT_CUDA(cub::DeviceSelect::Flagged(nullptr, b_sel, lkeys, lflags, cand + n_store, nsel, (int)n_live_box, s));
    KT_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, b_sort, cand, sorted, (int)ncand, 0, 63, s));
    KT_CUDA(cub::DeviceSelect::Unique(nullptr, b_uniq, sorted, uniq, nsel + 1, (int)ncand, s));
    const size_t tb = std::max(b_sel, std::max(b_sort, b_uniq));
    if (mem.device(&tmp, tb, who)) return KT_ERR_CUDA;
    size_t have = tb;
    KT_CUDA(cub::DeviceSelect::Flagged(tmp, have, lkeys, lflags, cand + n_store, nsel, (int)n_live_box, s));
    int n_live = 0;
    KT_CUDA(cudaMemcpyAsync(&n_live, nsel, sizeof(int), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const size_t nc = n_store + (size_t)n_live;
    int n_uniq = 0;
    if (nc) {
        have = tb;
        KT_CUDA(cub::DeviceRadixSort::SortKeys(tmp, have, cand, sorted, (int)nc, 0, 63, s));
        have = tb;
        KT_CUDA(cub::DeviceSelect::Unique(tmp, have, sorted, uniq, nsel + 1, (int)nc, s));
        KT_CUDA(cudaMemcpyAsync(&n_uniq, nsel + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
        KT_CUDA(cudaStreamSynchronize(s));
    }
    int16_t* mt = nullptr; uint8_t* mc = nullptr;
    if (mem.device(&mt, (size_t)n_uniq * MAPVOL_BRICK_VOXELS, who) || mem.device(&mc, (size_t)n_uniq * MAPVOL_BRICK_VOXELS * 4, who)) return KT_ERR_CUDA;
    if (n_uniq) {
        merge_bricks_kernel<<<(unsigned int)n_uniq, BRICK_THREADS, 0, s>>>(L, v, n_store > 0, uniq, mt, (uchar4*)mc);
        KT_LAUNCH_CHECK();
    }
    KT_CUDA(cudaEventRecord(ev[1], s));
    BrickSet set = {uniq, mt, mc, (size_t)n_uniq};
    float ms[3] = {0, 0, 0};
    if ((r = mesh_bricks(set, volume_size, vol, weight_cull, out, n_verts, n_tris, ms, s))) return r;
    if (rep) {
        std::memset(rep, 0, sizeof(*rep));
        rep->bricks = (size_t)n_uniq; rep->store_bricks = n_store; rep->live_bricks = (size_t)n_live;
        rep->input_voxels = (size_t)n_uniq * MAPVOL_BRICK_VOXELS; rep->output_verts = *n_verts; rep->output_tris = *n_tris;
        rep->store_full = full;
        KT_CUDA(cudaEventElapsedTime(&rep->gather_ms, ev[0], ev[1]));
        rep->mesh_ms = ms[0]; rep->sort_ms = ms[1]; rep->total_ms = rep->gather_ms + ms[2];
    }
    return 0;
}

} // namespace kt
