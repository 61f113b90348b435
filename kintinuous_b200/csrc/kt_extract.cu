// kintinuous_b200 -- zero-crossing point extraction from a slab of the cyclic TSDF volume.
//
// Replaces (reference, src/frontend/cuda/extract.cu): FullScan6Slice / extractKernelSlice / extractCloudSlice
// (:79-419), called through TsdfVolume::fetchCloud (TSDFVolume.cpp:131-172).
// Semantics kept: a voxel (W != 0, F != 1) emits one point per +x / +y / +z neighbour (W_n != 0, F_n != 1) whose
// TSDF has the strictly opposite sign; the point is the |F|-weighted mean of the two voxel centres, carries the
// NEIGHBOUR's colour with r/b swapped and this voxel's weight as alpha (Q8), and is shifted by
// realVoxelWrap*cell - size/2 (:310-312).  The +z neighbour is not range-checked: at z = V-1 it wraps to logical
// plane 0 through the cyclic addressing (Q12).  Point order is unspecified in the reference too (global atomicAdd).
// Design: the box is walked in STORAGE-contiguous order (x fastest) by a grid sized to the SM count, compaction
// is a warp-level prefix (shuffles + one atomicAdd per warp), points are written as two 16-byte stores, and -- unlike
// the reference (extract.cu:268-288) -- nothing is ever written past the caller's capacity.
// Bound: HBM, 6 B per slab voxel + 32 B per point.
#include "kt_ops.h"

namespace kt {

namespace {

struct ExtractParams {
    const int16_t* tsdf; const uchar4* color; int V; int3 wrap; int3 real_wrap; float3 cell;
    VolumeView vv; int multi;                              // shared volume: emit only for voxels of the storage planes this rank owns
    int minX, maxX, minY, maxY, minZ, maxZ, subsample;
    uint4* out; unsigned int capacity; unsigned int* counter;
};

__device__ __forceinline__ size_t vox_addr(const ExtractParams& p, int x, int y, int z)
{
    int sx = (x + p.wrap.x) % p.V, sy = (y + p.wrap.y) % p.V, sz = (z + p.wrap.z) % p.V;
    return ((size_t)sz * p.V + sy) * p.V + sx;
}

__device__ __forceinline__ float fetch(const ExtractParams& p, int x, int y, int z, int& weight, uchar4& c)
{
    if (p.multi) {
        // TSDF from the local replica; colour / weight from the plane's owner (local memory or NVLink peer)
        const int sx = (x + p.wrap.x) % p.V, sy = (y + p.wrap.y) % p.V, sz = (z + p.wrap.z) % p.V;
        float tsdf = unpack_tsdf(__ldg(&p.tsdf[((size_t)sz * p.V + sy) * p.V + sx]));
        const size_t a = ((size_t)vv_local_plane(p.vv, sz) * p.V + sy) * p.V + sx;
        c = __ldg(reinterpret_cast<const uchar4*>(p.vv.color[vv_owner(p.vv, sz)]) + a);
        weight = c.w;
        return tsdf;
    }
    size_t a = vox_addr(p, x, y, z);
    float tsdf = unpack_tsdf(__ldg(&p.tsdf[a]));
    c = __ldg(&p.color[a]);
    weight = c.w;
    return tsdf;
}

// (V * |Fn| + Vn * |F|) * d_inv with the contraction the reference build has (extract.cu:155, checked in its SASS:
// FMUL V*|Fn|; FFMA |F|*Vn + that; FMUL by the reciprocal).  Left to the compiler, the choice of which product is fused
// changes with unrelated edits and moves the point by 1 ulp.
__device__ __forceinline__ float interp(float V, float Vn, float F, float Fn, float d_inv)
{
    return __fmul_rn(__fmaf_rn(fabsf(F), Vn, __fmul_rn(V, fabsf(Fn))), d_inv);
}

__device__ __forceinline__ void store_point(const ExtractParams& p, unsigned int slot, float x, float y, float z, uchar4 ncol, int W)
{
    if (slot >= p.capacity) return;
    float px = x + p.real_wrap.x * p.cell.x - ((p.cell.x * p.V) / 2);
    float py = y + p.real_wrap.y * p.cell.y - ((p.cell.y * p.V) / 2);
    float pz = z + p.real_wrap.z * p.cell.z - ((p.cell.z * p.V) / 2);
    // PointXYZRGB bytes 16..19 are {b, g, r, a}; the reference stores r<-b, b<-r of the packed colour (Q8),
    // i.e. byte b = colour.x, byte g = colour.y, byte r = colour.z, byte a = W.
    unsigned int rgba = (unsigned int)ncol.x | ((unsigned int)ncol.y << 8) | ((unsigned int)ncol.z << 16) | ((unsigned int)(W & 0xff) << 24);
    uint4 lo = make_uint4(__float_as_uint(px), __float_as_uint(py), __float_as_uint(pz), 0u);
    uint4 hi = make_uint4(rgba, 0u, 0u, 0u);
    p.out[(size_t)slot * 2] = lo;
    p.out[(size_t)slot * 2 + 1] = hi;
}

__global__ void __launch_bounds__(256)
extract_kernel(const ExtractParams p)
{
    const int nx = p.maxX - p.minX, ny = p.maxY - p.minY, nz = p.maxZ - p.minZ;
    const size_t total = (size_t)nx * ny * nz;
    const size_t total_round = (total + 31) / 32 * 32;        // whole warps run the loop so the shuffles are convergent
    const unsigned int lane = threadIdx.x & 31;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total_round; idx += (size_t)gridDim.x * blockDim.x) {
        float4 pts[3]; uchar4 cols[3];
        int local_count = 0, W = 0;
        if (idx < total) {
            const int x = p.minX + (int)(idx % nx);
            const size_t r = idx / nx;
            const int y = p.minY + (int)(r % ny);
            const int z = p.minZ + (int)(r / ny);
            bool mine = true;
            if (p.multi) { const int sz = (z + p.wrap.z) % p.V; mine = vv_owner(p.vv, sz) == p.vv.rank; }
            if (mine && x < p.V && y < p.V && x % p.subsample == 0 && y % p.subsample == 0 && (z - p.minZ) % p.subsample == 0) {
                uchar4 c;
                float F = fetch(p, x, y, z, W, c);
                if (W != 0 && F != 1.f) {
                    float3 Vc;
                    Vc.x = (x + 0.5f) * p.cell.x; Vc.y = (y + 0.5f) * p.cell.y; Vc.z = (z + 0.5f) * p.cell.z;
                    if (x + 1 < p.V) {
                        int Wn; uchar4 cn;
                        float Fn = fetch(p, x + 1, y, z, Wn, cn);
                        if (Wn != 0 && Fn != 1.f)
                            if ((F > 0 && Fn < 0) || (F < 0 && Fn > 0)) {
                                float4 q; q.y = Vc.y; q.z = Vc.z;
                                float Vnx = Vc.x + p.cell.x;
                                float d_inv = 1.f / (fabs(F) + fabs(Fn));
                                q.x = interp(Vc.x, Vnx, F, Fn, d_inv);
                                pts[local_count] = q; cols[local_count] = cn; ++local_count;
                            }
                    }
                    if (y + 1 < p.V) {
                        int Wn; uchar4 cn;
                        float Fn = fetch(p, x, y + 1, z, Wn, cn);
                        if (Wn != 0 && Fn != 1.f)
                            if ((F > 0 && Fn < 0) || (F < 0 && Fn > 0)) {
                                float4 q; q.x = Vc.x; q.z = Vc.z;
                                float Vny = Vc.y + p.cell.y;
                                float d_inv = 1.f / (fabs(F) + fabs(Fn));
                                q.y = interp(Vc.y, Vny, F, Fn, d_inv);
                                pts[local_count] = q; cols[local_count] = cn; ++local_count;
                            }
                    }
                    {   // +z: unguarded, wraps through the cyclic addressing (Q12)
                        int Wn; uchar4 cn;
                        float Fn = fetch(p, x, y, z + 1, Wn, cn);
                        if (Wn != 0 && Fn != 1.f)
                            if ((F > 0 && Fn < 0) || (F < 0 && Fn > 0)) {
                                float4 q; q.x = Vc.x; q.y = Vc.y;
                                float Vnz = Vc.z + p.cell.z;
                                float d_inv = 1.f / (fabs(F) + fabs(Fn));
                                q.z = interp(Vc.z, Vnz, F, Fn, d_inv);
                                pts[local_count] = q; cols[local_count] = cn; ++local_count;
                            }
                    }
                }
            }
        }
        // warp compaction: exclusive prefix of local_count, one atomicAdd per warp
        int incl = local_count;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += v; }
        const int total_warp = __shfl_sync(0xffffffffu, incl, 31);
        if (total_warp > 0) {
            unsigned int base = 0;
            if (lane == 0) base = atomicAdd(p.counter, (unsigned int)total_warp);
            base = __shfl_sync(0xffffffffu, base, 0);
            const unsigned int off = base + (unsigned int)(incl - local_count);
            for (int l = 0; l < local_count; ++l) store_point(p, off + l, pts[l].x, pts[l].y, pts[l].z, cols[l], W);
        }
    }
}

} // namespace

// counter_dev must be zeroed by the caller (stream-ordered) before the launch; after it, *counter_dev = number of
// crossings found, which can exceed capacity (the caller clamps, like output_count = min(size, global_count)).
int extract_slice(const int16_t* tsdf, const float3& volume_size, int vol, void* out, size_t capacity, const int3& wrap,
                  const uint8_t* color, int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int subsample,
                  const int3& real_wrap, unsigned int* counter_dev, cudaStream_t s)
{
    if (maxX <= minX || maxY <= minY || maxZ <= minZ) return 0;
    ExtractParams p;
    p.tsdf = tsdf; p.color = (const uchar4*)color; p.V = vol; p.wrap = wrap_mod3(wrap, vol); p.real_wrap = real_wrap;
    p.multi = 0; p.vv = single_volume(const_cast<int16_t*>(tsdf), const_cast<uint8_t*>(color), vol);
    p.cell = make_float3(volume_size.x / vol, volume_size.y / vol, volume_size.z / vol);
    p.minX = minX; p.maxX = maxX; p.minY = minY; p.maxY = maxY; p.minZ = minZ; p.maxZ = maxZ; p.subsample = subsample < 1 ? 1 : subsample;
    p.out = (uint4*)out; p.capacity = (unsigned int)capacity; p.counter = counter_dev;
    size_t total = (size_t)(maxX - minX) * (maxY - minY) * (maxZ - minZ);
    size_t blocks = (total + 255) / 256;
    int grid = (int)(blocks < (size_t)device_info().sm_count * 16 ? blocks : (size_t)device_info().sm_count * 16);
    extract_kernel<<<grid, 256, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

int extract_slice_mg(const VolumeView& vv, const float3& volume_size, int vol, void* out, size_t capacity, const int3& wrap,
                     int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int subsample,
                     const int3& real_wrap, unsigned int* counter_dev, cudaStream_t s)
{
    if (maxX <= minX || maxY <= minY || maxZ <= minZ) return 0;
    ExtractParams p;
    p.tsdf = vv.tsdf[vv.rank]; p.color = (const uchar4*)vv.color[vv.rank]; p.V = vol; p.wrap = wrap_mod3(wrap, vol); p.real_wrap = real_wrap;
    p.cell = make_float3(volume_size.x / vol, volume_size.y / vol, volume_size.z / vol);
    p.minX = minX; p.maxX = maxX; p.minY = minY; p.maxY = maxY; p.minZ = minZ; p.maxZ = maxZ; p.subsample = subsample < 1 ? 1 : subsample;
    p.out = (uint4*)out; p.capacity = (unsigned int)capacity; p.counter = counter_dev;
    p.vv = vv; p.multi = 1;
    size_t total = (size_t)(maxX - minX) * (maxY - minY) * (maxZ - minZ);
    size_t blocks = (total + 255) / 256;
    int grid = (int)(blocks < (size_t)device_info().sm_count * 16 ? blocks : (size_t)device_info().sm_count * 16);
    extract_kernel<<<grid, 256, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
