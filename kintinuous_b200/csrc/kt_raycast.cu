// kintinuous_b200 -- surface prediction: ray-cast the TSDF from the current pose and build the model
// vertex / normal pyramid in the same launch.
//
// Replaces (reference, src/frontend/cuda/):
//   raycast / RayCaster / rayCastKernel          ray_caster.cu:56-471
//   resizeVMap / resizeNMap (x3 levels)          maps.cu:225-308  (KintinuousTracker.cpp:892-899)
// Design: one CTA = a 16x8 pixel tile; after the march the tile's vertices / normals sit in shared
// memory and the 2x2 means of levels 1..3 (8x4, 4x2, 2x1 pixels per tile) are produced by the same CTA,
// which removes 6 launches + 6 cudaDeviceSynchronize per frame and the 12 MB re-read of the level-0 maps.
// Per-ray arithmetic (march step, trilinear taps, gradient normal) keeps the reference's expression
// order; the volume is read through the read-only path with cyclic addressing by compare-subtract.
// Bound: L2 / latency (scattered 2-byte reads, about 60-100 per ray); DESIGN.md section 3.5.
#include "kt_ops.h"
#include <cstdlib>

namespace kt {

namespace {

struct RayParams {
    Intr intr; Mat33 Rcurr; float3 tcurr; float time_step; float3 volume_size; float3 cell_size;
    const int16_t* volume; const uchar4* color_volume; int V; int3 wrap;
    float* vmap[LEVELS]; float* nmap[LEVELS]; uchar4* vmap_color; int rows, cols; int n_levels;
    int z_begin;            // storage-z offset of the local slab (0 on a single GPU)
    // multi-GPU
    VolumeView vv; int tile_row_begin; int n_out;
    float* peer_vmap[MAX_GPUS][LEVELS]; float* peer_nmap[MAX_GPUS][LEVELS]; uchar4* peer_vcol[MAX_GPUS];
};

// POW2: V is a power of two (cyclic wrap by mask, plane / row offsets by shift); IdxT: 32-bit voxel index when V^3 <= 2^31.
template <bool POW2, typename IdxT, bool MG = false>
struct Caster {
    const RayParams& p;
    int shift;
    __device__ __forceinline__ Caster(const RayParams& p_) : p(p_) { shift = POW2 ? (31 - __clz(p_.V)) : 0; }

    __device__ __forceinline__ IdxT addr(int x, int y, int z) const
    {
        if (POW2) {
            const int m = p.V - 1;
            const unsigned int sx = (x + p.wrap.x) & m, sy = (y + p.wrap.y) & m, sz = (z + p.wrap.z) & m;
            return ((((IdxT)sz << shift) | sy) << shift) | sx;
        }
        int sx = x + p.wrap.x; if (sx >= p.V) sx -= p.V;
        int sy = y + p.wrap.y; if (sy >= p.V) sy -= p.V;
        int sz = z + p.wrap.z; if (sz >= p.V) sz -= p.V;
        return ((IdxT)sz * p.V + sy) * p.V + sx;
    }
    // shared volume (MG): the TSDF is replicated, so the march and every trilinear TSDF tap read LOCAL memory exactly as on one GPU; only
    // the colour / weight planes are sharded (block-cyclic by storage z): local memory or an NVLink peer (CUDA IPC) through the table
    __device__ __forceinline__ short rawTsdf(int x, int y, int z) const
    {
        return __ldg(&p.volume[addr(x, y, z)]);
    }
    __device__ __forceinline__ float readTsdf(int x, int y, int z) const { return unpack_tsdf(rawTsdf(x, y, z)); }
    __device__ __forceinline__ uchar4 readColor(int x, int y, int z) const
    {
        if (MG) {
            const int m = p.V - 1;
            const unsigned int sx = (x + p.wrap.x) & m, sy = (y + p.wrap.y) & m, sz = (z + p.wrap.z) & m;
            const unsigned int lz = (unsigned int)vv_local_plane(p.vv, (int)sz);
            return __ldg(reinterpret_cast<const uchar4*>(p.vv.color[vv_owner(p.vv, (int)sz)]) + ((((size_t)lz << shift) | sy) << shift | sx));
        }
        return __ldg(&p.color_volume[addr(x, y, z)]);
    }

    __device__ __forceinline__ int3 getVoxel(float3 point) const
    {
        int vx = __float2int_rd(point.x / p.cell_size.x);
        int vy = __float2int_rd(point.y / p.cell_size.y);
        int vz = __float2int_rd(point.z / p.cell_size.z);
        return make_int3(vx, vy, vz);
    }
    __device__ __forceinline__ bool checkInds(const int3& g) const
    {
        return ((unsigned)g.x < (unsigned)p.V && (unsigned)g.y < (unsigned)p.V && (unsigned)g.z < (unsigned)p.V);
    }

    // trilinear weights and base voxel of a point; false if the base voxel is outside [1, V-2]
    __device__ __forceinline__ bool trilinearSetup(const float3& point, int3& g, float& a, float& b, float& c) const
    {
        g = getVoxel(point);
        if (g.x <= 0 || g.x >= p.V - 1) return false;
        if (g.y <= 0 || g.y >= p.V - 1) return false;
        if (g.z <= 0 || g.z >= p.V - 1) return false;
        float vx = (g.x + 0.5f) * p.cell_size.x;
        float vy = (g.y + 0.5f) * p.cell_size.y;
        float vz = (g.z + 0.5f) * p.cell_size.z;
        g.x = (point.x < vx) ? (g.x - 1) : g.x;
        g.y = (point.y < vy) ? (g.y - 1) : g.y;
        g.z = (point.z < vz) ? (g.z - 1) : g.z;
        a = __fmaf_rn(-(g.x + 0.5f), p.cell_size.x, point.x) / p.cell_size.x;        // (point.x - (g.x + 0.5f) * cell.x) / cell.x
        b = __fmaf_rn(-(g.y + 0.5f), p.cell_size.y, point.y) / p.cell_size.y;
        c = __fmaf_rn(-(g.z + 0.5f), p.cell_size.z, point.z) / p.cell_size.z;
        return true;
    }

    __device__ __forceinline__ float interpolateTrilineary(const float3& point) const
    {
        int3 g; float a, b, c;
        if (!trilinearSetup(point, g, a, b, c)) return qnan();
        float res = readTsdf(g.x + 0, g.y + 0, g.z + 0) * (1 - a) * (1 - b) * (1 - c) +
                    readTsdf(g.x + 0, g.y + 0, g.z + 1) * (1 - a) * (1 - b) * c +
                    readTsdf(g.x + 0, g.y + 1, g.z + 0) * (1 - a) * b * (1 - c) +
                    readTsdf(g.x + 0, g.y + 1, g.z + 1) * (1 - a) * b * c +
                    readTsdf(g.x + 1, g.y + 0, g.z + 0) * a * (1 - b) * (1 - c) +
                    readTsdf(g.x + 1, g.y + 0, g.z + 1) * a * (1 - b) * c +
                    readTsdf(g.x + 1, g.y + 1, g.z + 0) * a * b * (1 - c) +
                    readTsdf(g.x + 1, g.y + 1, g.z + 1) * a * b * c;
        return res;
    }

    // colour (r,g,b truncated to u8) and weight ("heat") trilinear taps share the 8 uchar4 loads
    __device__ __forceinline__ uchar4 interpolateColorHeat(const float3& point) const
    {
        int3 g; float a, b, c;
        if (!trilinearSetup(point, g, a, b, c)) {
            // interpolateColorTrilineary returns black, interpolateHeatTrilineary NaN -> (unsigned char)NaN
            uchar4 r; r.x = 0; r.y = 0; r.z = 0; r.w = (unsigned char)qnan();
            return r;
        }
        const uchar4 c000 = readColor(g.x + 0, g.y + 0, g.z + 0), c001 = readColor(g.x + 0, g.y + 0, g.z + 1);
        const uchar4 c010 = readColor(g.x + 0, g.y + 1, g.z + 0), c011 = readColor(g.x + 0, g.y + 1, g.z + 1);
        const uchar4 c100 = readColor(g.x + 1, g.y + 0, g.z + 0), c101 = readColor(g.x + 1, g.y + 0, g.z + 1);
        const uchar4 c110 = readColor(g.x + 1, g.y + 1, g.z + 0), c111 = readColor(g.x + 1, g.y + 1, g.z + 1);
#define KT_TRI(f) ((float)c000.f * (1 - a) * (1 - b) * (1 - c) + (float)c001.f * (1 - a) * (1 - b) * c + \
                   (float)c010.f * (1 - a) * b * (1 - c) + (float)c011.f * (1 - a) * b * c + \
                   (float)c100.f * a * (1 - b) * (1 - c) + (float)c101.f * a * (1 - b) * c + \
                   (float)c110.f * a * b * (1 - c) + (float)c111.f * a * b * c)
        uchar4 r;
        r.x = KT_TRI(x); r.y = KT_TRI(y); r.z = KT_TRI(z);
        float heat = KT_TRI(w);
        r.w = heat;
#undef KT_TRI
        return r;
    }
};

__device__ __forceinline__ float getMinTime(const float3& volume_max, const float3& origin, const float3& dir)
{
    float txmin = ((dir.x > 0 ? 0.f : volume_max.x) - origin.x) / dir.x;
    float tymin = ((dir.y > 0 ? 0.f : volume_max.y) - origin.y) / dir.y;
    float tzmin = ((dir.z > 0 ? 0.f : volume_max.z) - origin.z) / dir.z;
    return fmax(fmax(txmin, tymin), tzmin);
}
__device__ __forceinline__ float getMaxTime(const float3& volume_max, const float3& origin, const float3& dir)
{
    float txmax = ((dir.x > 0 ? volume_max.x : 0.f) - origin.x) / dir.x;
    float tymax = ((dir.y > 0 ? volume_max.y : 0.f) - origin.y) / dir.y;
    float tzmax = ((dir.z > 0 ? volume_max.z : 0.f) - origin.z) / dir.z;
    return fmin(fmin(txmax, tymax), tzmax);
}

// 16x8-pixel CTAs (a warp = 16x2 pixels): 2400 CTAs at 640x480 instead of 1200 halve the scheduling quantum of a launch that is only
// ~2 CTA rounds long (stage timer 72.8 -> 68.8 us against 32x8 tiles), and a 16x2 warp footprint keeps the rays of a warp closer.
enum { RC_X = 16, RC_Y = 8 };

// ray_start + ray_dir * t, as the fused multiply-add nvcc makes of the reference's expression (ray_caster.cu:337-411)
__device__ __forceinline__ float3 ray_at(const float3& o, const float3& d, float t)
{
    return make_float3(__fmaf_rn(d.x, t, o.x), __fmaf_rn(d.y, t, o.y), __fmaf_rn(d.z, t, o.z));
}

// One ray.  Returns validity of vertex / normal; outputs by reference.
template <bool POW2, typename IdxT, int RS, bool MG>
__device__ __forceinline__ void cast_ray(const RayParams& p, int x, int y, bool& v_ok, float3& vtx, bool& n_ok, float3& nrm,
                                         bool& c_ok, uchar4& col)
{
    v_ok = false; n_ok = false; c_ok = false;
    Caster<POW2, IdxT, MG> rc(p);
    float3 ray_start = p.tcurr;
    float3 ray_next_c;
    ray_next_c.x = (x - p.intr.cx) / p.intr.fx;
    ray_next_c.y = (y - p.intr.cy) / p.intr.fy;
    ray_next_c.z = 1;
    float3 ray_next = add3(mul33(p.Rcurr, ray_next_c), p.tcurr);
    float3 ray_dir = normalized3(sub3(ray_next, ray_start));
    ray_dir.x = (ray_dir.x == 0.f) ? 1e-15 : ray_dir.x;
    ray_dir.y = (ray_dir.y == 0.f) ? 1e-15 : ray_dir.y;
    ray_dir.z = (ray_dir.z == 0.f) ? 1e-15 : ray_dir.z;

    float time_start_volume = getMinTime(p.volume_size, ray_start, ray_dir);
    float time_exit_volume = getMaxTime(p.volume_size, ray_start, ray_dir);
    const float min_dist = 0.f;
    time_start_volume = fmax(time_start_volume, min_dist);
    if (time_start_volume >= time_exit_volume) return;

    const float time_step = p.time_step;
    float time_curr = time_start_volume;
    int3 g = rc.getVoxel(ray_at(ray_start, ray_dir, time_curr));
    g.x = max(0, min(g.x, p.V - 1));
    g.y = max(0, min(g.y, p.V - 1));
    g.z = max(0, min(g.z, p.V - 1));
    // the march only needs the SIGN of the TSDF, and sign(short / 32767) == sign(short) (no underflow: |1/32767| is normal)
    int tsdf = rc.rawTsdf(g.x, g.y, g.z);

    const float max_time = 3 * (p.volume_size.x + p.volume_size.y + p.volume_size.z);
    // The march (ray_caster.cu:345-425) is evaluated strictly in order, but the nearest-voxel reads of the next RS steps are
    // issued together: a step only needs the previous TSDF value to DECIDE, not to ADDRESS, so RS dependent L2 round trips
    // become one.  time_curr advances by the same sequence of float additions as the reference's for-loop.
    bool done = false;
    while (!done && time_curr < max_time) {
        float tq[RS]; bool inb[RS]; short raw[RS];
        float t = time_curr;
#pragma unroll
        for (int s = 0; s < RS; ++s) {
            tq[s] = t;
            int3 gn = rc.getVoxel(ray_at(ray_start, ray_dir, (t + time_step)));
            inb[s] = rc.checkInds(gn);
            raw[s] = inb[s] ? rc.rawTsdf(gn.x, gn.y, gn.z) : (short)0;
            t += time_step;
        }
#pragma unroll
        for (int s = 0; s < RS; ++s) {
            if (done) break;
            const float tc = tq[s];
            if (!(tc < max_time)) { done = true; break; }
            const int tsdf_prev = tsdf;
            if (!inb[s]) { done = true; break; }
            tsdf = raw[s];
            if (tsdf_prev < 0 && tsdf > 0) { done = true; break; }
            if (tsdf_prev > 0 && tsdf < 0) {
                done = true;
                float Ftdt = rc.interpolateTrilineary(ray_at(ray_start, ray_dir, (tc + time_step)));
                if (isnan(Ftdt)) break;
                float Ft = rc.interpolateTrilineary(ray_at(ray_start, ray_dir, tc));
                if (isnan(Ft)) break;

                float Ts = tc - time_step * Ft / (Ftdt - Ft);
                float3 vetex_found = ray_at(ray_start, ray_dir, Ts);
                vtx = vetex_found; v_ok = true;

                int3 gc = rc.getVoxel(ray_at(ray_start, ray_dir, tc));
                col = rc.interpolateColorHeat(vetex_found); c_ok = true;

                if (gc.x > 1 && gc.y > 1 && gc.z > 1 && gc.x < p.V - 2 && gc.y < p.V - 2 && gc.z < p.V - 2) {
                    float3 tt, n;
                    tt = vetex_found; tt.x += p.cell_size.x; float Fx1 = rc.interpolateTrilineary(tt);
                    tt = vetex_found; tt.x -= p.cell_size.x; float Fx2 = rc.interpolateTrilineary(tt);
                    n.x = (Fx1 - Fx2);
                    tt = vetex_found; tt.y += p.cell_size.y; float Fy1 = rc.interpolateTrilineary(tt);
                    tt = vetex_found; tt.y -= p.cell_size.y; float Fy2 = rc.interpolateTrilineary(tt);
                    n.y = (Fy1 - Fy2);
                    tt = vetex_found; tt.z += p.cell_size.z; float Fz1 = rc.interpolateTrilineary(tt);
                    tt = vetex_found; tt.z -= p.cell_size.z; float Fz2 = rc.interpolateTrilineary(tt);
                    n.z = (Fz1 - Fz2);
                    nrm = normalized3(n); n_ok = true;
                }
                break;
            }
        }
        time_curr = t;
    }
}

// 2x2 mean of one pyramid step inside the CTA (maps.cu:225-277): in/out are [3][H][W] tiles in smem.
template <bool normalize>
__device__ __forceinline__ bool resize_tile(const float* in, int W, int H, int ox, int oy, float3& out)
{
    const int xs = ox * 2, ys = oy * 2;
    const int plane = W * H;
    float x00 = in[ys * W + xs], x01 = in[ys * W + xs + 1], x10 = in[(ys + 1) * W + xs], x11 = in[(ys + 1) * W + xs + 1];
    if (isnan(x00) || isnan(x01) || isnan(x10) || isnan(x11)) return false;
    float3 n;
    n.x = (x00 + x01 + x10 + x11) / 4;
    const float* iy = in + plane;
    n.y = (iy[ys * W + xs] + iy[ys * W + xs + 1] + iy[(ys + 1) * W + xs] + iy[(ys + 1) * W + xs + 1]) / 4;
    const float* iz = in + 2 * plane;
    n.z = (iz[ys * W + xs] + iz[ys * W + xs + 1] + iz[(ys + 1) * W + xs] + iz[(ys + 1) * W + xs + 1]) / 4;
    if (normalize) n = normalized3(n);
    out = n;
    return true;
}

// store one pyramid-level sample into the model maps of every destination (1 locally; all ranks when sharded: the
// all-gather of the predicted surface is these P2P stores)
template <bool MG>
__device__ __forceinline__ void store_maps(const RayParams& p, int level, size_t i, size_t P, bool okv, const float3& v, bool okn, const float3& n)
{
    const float nan = qnan();
    const int n_out = MG ? p.n_out : 1;
    for (int g = 0; g < n_out; ++g) {
        float* vm = MG ? p.peer_vmap[g][level] : p.vmap[level];
        float* nm = MG ? p.peer_nmap[g][level] : p.nmap[level];
        if (okv) { vm[i] = v.x; vm[i + P] = v.y; vm[i + 2 * P] = v.z; } else vm[i] = nan;
        if (okn) { nm[i] = n.x; nm[i + P] = n.y; nm[i + 2 * P] = n.z; } else nm[i] = nan;
    }
}

template <bool POW2, typename IdxT, int RS, int MINB, bool MG>
__global__ void __launch_bounds__(RC_X * RC_Y, MINB)
raycast_kernel(const RayParams p)
{
    // level-0 tile, then levels 1..3 (each [v|n][3 planes][H][W])
    __shared__ float s0[2][3][RC_Y][RC_X];
    __shared__ float s1[2][3][RC_Y / 2][RC_X / 2];
    __shared__ float s2[2][3][RC_Y / 4][RC_X / 4];

    const int tile_y = blockIdx.y + (MG ? p.tile_row_begin : 0);
    const int x = threadIdx.x + blockIdx.x * RC_X;
    const int y = threadIdx.y + tile_y * RC_Y;
    const float nan = qnan();
    const bool inside = (x < p.cols && y < p.rows);

    bool v_ok = false, n_ok = false, c_ok = false;
    float3 vtx = make_float3(nan, nan, nan), nrm = make_float3(nan, nan, nan);
    uchar4 col;
    if (inside) {
        cast_ray<POW2, IdxT, RS, MG>(p, x, y, v_ok, vtx, n_ok, nrm, c_ok, col);
        const size_t P = (size_t)p.rows * p.cols, i = (size_t)y * p.cols + x;
        // like the reference: x planes are always written (NaN = no surface), y/z only on success
        store_maps<MG>(p, 0, i, P, v_ok, vtx, n_ok, nrm);
        if (c_ok) { if (MG) { for (int g = 0; g < p.n_out; ++g) p.peer_vcol[g][i] = col; } else p.vmap_color[i] = col; }
    }
    if (p.n_levels <= 1) return;

    s0[0][0][threadIdx.y][threadIdx.x] = v_ok ? vtx.x : nan; s0[0][1][threadIdx.y][threadIdx.x] = vtx.y; s0[0][2][threadIdx.y][threadIdx.x] = vtx.z;
    s0[1][0][threadIdx.y][threadIdx.x] = n_ok ? nrm.x : nan; s0[1][1][threadIdx.y][threadIdx.x] = nrm.y; s0[1][2][threadIdx.y][threadIdx.x] = nrm.z;
    __syncthreads();

    // level 1: RC_X/2 x RC_Y/2 outputs per tile
    {
        const int W = RC_X / 2, H = RC_Y / 2;
        const int rows1 = p.rows >> 1, cols1 = p.cols >> 1;
        if (threadIdx.x < W && threadIdx.y < H) {
            const int ox = threadIdx.x, oy = threadIdx.y;
            const int gx = blockIdx.x * W + ox, gy = tile_y * H + oy;
            float3 v, n;
            bool okv = resize_tile<false>(&s0[0][0][0][0], RC_X, RC_Y, ox, oy, v);
            bool okn = resize_tile<true>(&s0[1][0][0][0], RC_X, RC_Y, ox, oy, n);
            s1[0][0][oy][ox] = okv ? v.x : nan; s1[0][1][oy][ox] = v.y; s1[0][2][oy][ox] = v.z;
            s1[1][0][oy][ox] = okn ? n.x : nan; s1[1][1][oy][ox] = n.y; s1[1][2][oy][ox] = n.z;
            if (gx < cols1 && gy < rows1) {
                const size_t P = (size_t)rows1 * cols1, i = (size_t)gy * cols1 + gx;
                store_maps<MG>(p, 1, i, P, okv, v, okn, n);
            }
        }
    }
    if (p.n_levels <= 2) return;
    __syncthreads();
    {
        const int W = RC_X / 4, H = RC_Y / 4;
        const int rows2 = p.rows >> 2, cols2 = p.cols >> 2;
        if (threadIdx.x < W && threadIdx.y < H) {
            const int ox = threadIdx.x, oy = threadIdx.y;
            const int gx = blockIdx.x * W + ox, gy = tile_y * H + oy;
            float3 v, n;
            bool okv = resize_tile<false>(&s1[0][0][0][0], RC_X / 2, RC_Y / 2, ox, oy, v);
            bool okn = resize_tile<true>(&s1[1][0][0][0], RC_X / 2, RC_Y / 2, ox, oy, n);
            s2[0][0][oy][ox] = okv ? v.x : nan; s2[0][1][oy][ox] = v.y; s2[0][2][oy][ox] = v.z;
            s2[1][0][oy][ox] = okn ? n.x : nan; s2[1][1][oy][ox] = n.y; s2[1][2][oy][ox] = n.z;
            if (gx < cols2 && gy < rows2) {
                const size_t P = (size_t)rows2 * cols2, i = (size_t)gy * cols2 + gx;
                store_maps<MG>(p, 2, i, P, okv, v, okn, n);
            }
        }
    }
    if (p.n_levels <= 3) return;
    __syncthreads();
    {
        const int W = RC_X / 8, H = RC_Y / 8;
        const int rows3 = p.rows >> 3, cols3 = p.cols >> 3;
        if (threadIdx.x < W && threadIdx.y < H) {
            const int ox = threadIdx.x, oy = threadIdx.y;
            const int gx = blockIdx.x * W + ox, gy = tile_y * H + oy;
            float3 v, n;
            bool okv = resize_tile<false>(&s2[0][0][0][0], RC_X / 4, RC_Y / 4, ox, oy, v);
            bool okn = resize_tile<true>(&s2[1][0][0][0], RC_X / 4, RC_Y / 4, ox, oy, n);
            if (gx < cols3 && gy < rows3) {
                const size_t P = (size_t)rows3 * cols3, i = (size_t)gy * cols3 + gx;
                store_maps<MG>(p, 3, i, P, okv, v, okn, n);
            }
        }
    }
}

} // namespace

int raycast(const RaycastArgs& a, cudaStream_t s)
{
    RayParams p;
    p.intr = a.k; p.Rcurr = a.R; p.tcurr = a.t; p.time_step = a.trunc * 0.8f; p.volume_size = a.volume_size;
    p.cell_size = make_float3(a.volume_size.x / a.vol, a.volume_size.y / a.vol, a.volume_size.z / a.vol);
    p.volume = a.tsdf; p.color_volume = (const uchar4*)a.color; p.V = a.vol; p.wrap = wrap_mod3(a.wrap, a.vol);
    for (int l = 0; l < LEVELS; ++l) { p.vmap[l] = a.vmap[l]; p.nmap[l] = a.nmap[l]; }
    p.vmap_color = (uchar4*)a.vmap_color; p.rows = a.rows; p.cols = a.cols;
    p.n_levels = a.n_levels; p.z_begin = 0; p.tile_row_begin = 0; p.n_out = 1;
    // the in-tile pyramid needs every level's tile to be whole
    if (p.n_levels > 1 && ((a.cols % RC_X) != 0 || (a.rows % RC_Y) != 0)) { set_error("raycast: fused pyramid needs cols %% 16 == 0 and rows %% 8 == 0"); return -1; }
    dim3 block(RC_X, RC_Y), grid(div_up(a.cols, RC_X), div_up(a.rows, RC_Y));
    const bool pow2 = (a.vol & (a.vol - 1)) == 0;
    static const bool force64 = getenv("KT_FORCE_IDX64") != nullptr;     // test hook, see kt_tsdf.cu
    const bool idx32 = !force64 && (size_t)a.vol * a.vol * a.vol <= ((size_t)1 << 31);
    if (a.multi) {
        if (!pow2) { set_error("raycast: the shared volume needs a power-of-two resolution"); return -1; }
        p.vv = a.vv; p.tile_row_begin = a.tile_row_begin; p.n_out = a.vv.world;
        p.volume = a.vv.tsdf[a.vv.rank];                      // the local TSDF replica
        for (int g = 0; g < MAX_GPUS; ++g) { for (int l = 0; l < LEVELS; ++l) { p.peer_vmap[g][l] = a.peer_vmap[g][l]; p.peer_nmap[g][l] = a.peer_nmap[g][l]; } p.peer_vcol[g] = (uchar4*)a.peer_vcol[g]; }
        grid.y = a.tile_row_end - a.tile_row_begin;
        if (grid.y > 0) {
            if (idx32) raycast_kernel<true, unsigned int, 8, 8, true><<<grid, block, 0, s>>>(p);
            else raycast_kernel<true, size_t, 8, 8, true><<<grid, block, 0, s>>>(p);
        }
    }
    else if (pow2 && idx32) {
        // 8 speculative steps per batch at 8 CTAs/SM (4 steps per batch and 10 CTAs/SM, which spills, were slower)
        raycast_kernel<true, unsigned int, 8, 8, false><<<grid, block, 0, s>>>(p);
    }
    else if (pow2) raycast_kernel<true, size_t, 8, 8, false><<<grid, block, 0, s>>>(p);
    else if (idx32) raycast_kernel<false, unsigned int, 8, 8, false><<<grid, block, 0, s>>>(p);
    else raycast_kernel<false, size_t, 8, 8, false><<<grid, block, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
