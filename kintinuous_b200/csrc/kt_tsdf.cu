// kintinuous_b200 -- TSDF volume: initialise, clear shifted-out slabs, integrate a depth frame.
//
// Replaces (reference, src/frontend/cuda/tsdf_volume.cu):
//   initVolume / initColorVolume                         :452-479, :57-86
//   clearVolume{X,Y,Z}[Back][c] (12 wrappers, 6 kernels) :88-448
//   scaleDepth                                           :491-538   (fused with the bilateral filter: kt_pyramid.cu, bilateral_scale_kernel)
//   tsdf23 / integrateTsdfVolume                         :541-674
// Volume layout (DESIGN.md section 2): two planes in HBM, exactly the reference's encoding so that
// kt_volume_export_reference_layout is a plain copy: tsdf short[V^3] (value * 32767, round toward zero)
// and colour uchar4[V^3] = {r, g, b, weight}; x fastest; cyclic ("shifting") addressing
//   storage(x,y,z) = ((x+wx)%V) + ((y+wy)%V)*V + ((z+wz)%V)*V^2        (tsdf_volume.cu:612)
// Re-layout of the WORK, not of the bytes: threads are mapped to STORAGE coordinates (the
// reference maps them to logical coordinates, so after a shift every warp straddles sector
// boundaries); a warp always owns one aligned 64-B tsdf segment + one aligned 128-B colour line per z,
// the z axis is split into 16 chunks (grid.z) for 16x more CTAs than the reference's 1 024, whole columns
// and z-ranges outside the view frustum are skipped analytically (about 95 % of a centred 6 m cube),
// and slab clears / init use 128-bit stores.
// Exactness: the reference advances v_x, v_y, v_g_z, z_scaled by repeated float additions along z
// (:565-574); rounding of those running sums decides which depth pixel a voxel reads, so the same
// sequence of additions is replayed here (the z tables once per launch, v_x / v_y per thread).
// The colour update's per-pixel half (normal validity, view-angle weight, RGB as float) is prepared once per frame (color_prep_kernel).
// Roofline: HBM by nature (12 B per updated voxel + image-side gathers), instruction-issue bound in practice (DESIGN.md section 4).
#include "kt_ops.h"
#include "kt_replay.cuh"
#include "kt_frustum.hpp"

namespace kt {

namespace {

// ------------------------------------------------------------------------------------------------
// fills
__global__ void __launch_bounds__(256) fill_zero_u4(uint4* __restrict__ p, size_t n16)
{
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) p[i] = z;
}

// Clear `count` consecutive storage planes [p0, p0+count) (mod V) along `axis` in both volumes.
// Work item = 8 consecutive x voxels (16 B of tsdf, 32 B of colour) for the y / z axes.
// Shared volume (vv.world > 1): the TSDF planes of the local replica are all cleared here (every rank clears its own replica, no
// traffic), the colour planes only where this rank owns the storage z plane.
__global__ void __launch_bounds__(256)
clear_planes_yz_kernel(int16_t* __restrict__ tsdf, uint8_t* __restrict__ color, int V, int axis, int p0, int count, const VolumeView vv)
{
    const int xg = V / 8;                                   // groups of 8 voxels per row
    const size_t total = (size_t)count * V * xg;
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        int g = (int)(idx % xg);
        size_t r = idx / xg;
        int other = (int)(r % V);
        int i = (int)(r / V);
        int plane = p0 + i; if (plane >= V) plane -= V;
        int sy = axis == 1 ? plane : other;
        int sz = axis == 1 ? other : plane;
        *reinterpret_cast<uint4*>(tsdf + ((size_t)sz * V + sy) * V + (size_t)g * 8) = z4;
        if (vv_owner(vv, sz) != vv.rank) continue;            // not this rank's colour plane
        size_t base = ((size_t)vv_local_plane(vv, sz) * V + sy) * V + (size_t)g * 8;
        uint4* c = reinterpret_cast<uint4*>(color + base * 4);
        c[0] = z4; c[1] = z4;
    }
}

__global__ void __launch_bounds__(256)
clear_planes_x_kernel(int16_t* __restrict__ tsdf, uchar4* __restrict__ color, int V, int p0, int count, const VolumeView vv)
{
    const size_t total = (size_t)count * V * V;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        int i = (int)(idx % count);
        size_t r = idx / count;                              // r = sz * V + sy
        int sx = p0 + i; if (sx >= V) sx -= V;
        const int sz = (int)(r / V), sy = (int)(r - (size_t)sz * V);
        tsdf[r * V + sx] = 0;
        if (vv_owner(vv, sz) != vv.rank) continue;
        color[((size_t)vv_local_plane(vv, sz) * V + sy) * V + sx] = make_uchar4(0, 0, 0, 0);
    }
}

// ------------------------------------------------------------------------------------------------
// z tables: v_g_z(z) and z_scaled(z) as the reference's running sums produce them (tsdf_volume.cu:555,563,570-571: they start at
// (0 + 0.5f) * cell - t_z and 0 and grow by ONE float addition of cell per z step).  Prologue of the integration, one small launch: entry
// z is brought there by thread z with the exact fast-forward of kt_replay.cuh (round 1: one thread adding 2 V times, 6 us on the critical
// path between the odometry and the integration; building the entries inside integrate_kernel -- per thread, or per CTA in shared
// memory -- was slower in the design's measurements), and the other job of this launch is the reset of the odometry
// kernels' exchange words for the next frame (grid_sum_words, kt_frame.cuh): it sits between two odometry launches anyway.
__global__ void __launch_bounds__(256) ztable_kernel(float* __restrict__ table, int V, float cell_z, float t_z, unsigned long long* __restrict__ reset_words, int reset_count, int reset_stride, int seq)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (blockIdx.x == 0) for (int k = threadIdx.x; k < reset_count; k += blockDim.x) reset_words[(size_t)k * reset_stride] = 0ull;
    if (i >= 2 * V) return;
    const int z = i < V ? i : i - V;
    float v = i < V ? __fmaf_rn(0.5f, cell_z, -t_z) : 0.f;                 // (0 + 0.5f) * cell_z - t_z (0.5 * cell is exact, so fused or not is the same)
    if (seq) { for (int k = 0; k < z; ++k) v = __fadd_rn(v, cell_z); }    // KT_INT_SEQ_REPLAY (test hook): the additions one by one
    else v = replay_add(v, cell_z, z);
    table[i] = v;
}

struct IntegrateParams {
    const float* depth_scaled; int rows, cols; Intr k; float3 cell; Mat33 Rinv; float3 t; float trunc;
    int16_t* tsdf; uchar4* color; int V; int3 wrap; const uint8_t* rgb; const float* nmap; bool angle_color;
    const float* ztable; int zchunk;
    const float* cw; const float4* rgbf;   // PREP: per-pixel colour weight (sign bit = normal invalid) and RGB as floats
    int lz_lo, lz_hi;          // LOGICAL z range walked by this launch
    int z_far_first;           // schedule the z chunks from high z to low z (see integrate())
    VolumeView vv;             // shared volume (MG instances): plane ownership and the peers' TSDF replicas
    int seq_replay;            // test hook: replay the running sums one addition at a time instead of replay_add()
    int mg_no_publish;         // KT_MG_NO_PUBLISH (diagnostic only, results are wrong): skip the P2P stores of changed TSDF values
    int tile_x0, tiles_x, tile_y0, tiles_y;    // the launch covers the cyclic range of 32-wide / 8-high storage tiles [tile0, tile0 + gridDim) mod tiles (kt_frustum.hpp)
};

#define KT_MAX_WEIGHT 128          // Tsdf::MAX_WEIGHT (tsdf_volume.cu:486)
#define KT_RGB_VIEW_ANGLE_WEIGHT 0.75f

// Per-pixel part of the colour update, once per frame instead of once per voxel (tsdf_volume.cu:601-622): the view-angle weight
// Wrkc = min(1, |n_z| / 0.75) * 2 (or 2 without angle weighting) depends only on the pixel; its sign bit carries isnan(n_x).  RGB is
// widened to float (exact).  The voxel loop then needs 2 loads (4 B + 16 B) instead of 5 and no per-voxel conversion of the image.
__global__ void __launch_bounds__(256)
color_prep_kernel(const float* __restrict__ nmap, const uchar3* __restrict__ rgb, int n, bool angle_color, float* __restrict__ cw, float4* __restrict__ rgbf)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float nx = nmap[i];
    float nz = nmap[i + 2 * (size_t)n];
    if (nz < 0) nz = -nz;
    const float Wrkc = (angle_color ? min(1.0f, nz / KT_RGB_VIEW_ANGLE_WEIGHT) : 1.0f) * 2.0f;
    cw[i] = isnan(nx) ? -Wrkc : Wrkc;
    const uchar3 c = rgb[i];
    rgbf[i] = make_float4((float)c.x, (float)c.y, (float)c.z, 0.f);
}

__device__ __forceinline__ unsigned int sat_u8_rn(float x)       // == min(255, max(0, __float2int_rn(x))), one instruction
{
    unsigned int r;
    asm("cvt.rni.sat.u8.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// MG: the volume is shared by vv.world GPUs (VolumeView, kt_ops.h): this launch updates only the voxels of storage planes this rank owns
// -- it steps over the foreign blocks of planes -- and stores every CHANGED TSDF value into all ranks' replicas.
template <typename IdxT, int ZU, int MINB, bool PREP = false, bool MG = false>
__global__ void __launch_bounds__(256, MINB)
integrate_kernel(const IntegrateParams p)
{
    const int V = p.V;
    int bx = p.tile_x0 + (int)blockIdx.x; if (bx >= p.tiles_x) bx -= p.tiles_x;      // the grid spans only the frustum's box of storage tiles (cyclic)
    int by = p.tile_y0 + (int)blockIdx.y; if (by >= p.tiles_y) by -= p.tiles_y;
    const int sx = bx * 32 + threadIdx.x;          // STORAGE x, y
    const int sy = by * 8 + threadIdx.y;
    const int z0 = p.lz_lo + (p.z_far_first ? (int)(gridDim.z - 1 - blockIdx.z) : (int)blockIdx.z) * p.zchunk;
    const int z1 = min(z0 + p.zchunk, p.lz_hi);

    const float3 cell_size = p.cell;
    const Intr intr = p.k;
    const Mat33 Rcurr_inv = p.Rinv;
    const float3 tcurr = p.t;
    const float tranc_dist = p.trunc;
    const int cols = p.cols, rows = p.rows;

    if (sx >= V || sy >= V) return;
    int x = sx - p.wrap.x; if (x < 0) x += V;             // logical voxel
    int y = sy - p.wrap.y; if (y < 0) y += V;

    // Parity-critical arithmetic is written with explicit round-to-nearest intrinsics in exactly the contraction nvcc chose for the
    // reference's expressions (tsdf_volume.cu:549-563; read off the SASS of both builds): a*b + c*d compiles to fma(a, b, c*d).  Left to
    // the compiler, an unrelated edit of this kernel can flip which product is fused and move a voxel's projection by one ulp.
    float v_g_x = __fmaf_rn(x + 0.5f, cell_size.x, -tcurr.x);                            // (x + 0.5f) * cell_size.x - tcurr.x
    float v_g_y = __fmaf_rn(y + 0.5f, cell_size.y, -tcurr.y);
    float v_g_z = __fmaf_rn(0.5f, cell_size.z, -tcurr.z);                                // (0 + 0.5f) * cell_size.z - tcurr.z

    float v_g_part_norm = __fmaf_rn(v_g_x, v_g_x, __fmul_rn(v_g_y, v_g_y));              // v_g_x * v_g_x + v_g_y * v_g_y

    // (R.x * v_g_x + R.y * v_g_y + R.z * v_g_z) [* f]
    float v_x = __fmul_rn(__fmaf_rn(Rcurr_inv.r0.z, v_g_z, __fmaf_rn(Rcurr_inv.r0.x, v_g_x, __fmul_rn(Rcurr_inv.r0.y, v_g_y))), intr.fx);
    float v_y = __fmul_rn(__fmaf_rn(Rcurr_inv.r1.z, v_g_z, __fmaf_rn(Rcurr_inv.r1.x, v_g_x, __fmul_rn(Rcurr_inv.r1.y, v_g_y))), intr.fy);
    float v_z = __fmaf_rn(Rcurr_inv.r2.z, v_g_z, __fmaf_rn(Rcurr_inv.r2.x, v_g_x, __fmul_rn(Rcurr_inv.r2.y, v_g_y)));

    float Rcurr_inv_0_z_scaled = Rcurr_inv.r0.z * cell_size.z * intr.fx;      // used by the conservative frustum interval only
    float Rcurr_inv_1_z_scaled = Rcurr_inv.r1.z * cell_size.z * intr.fy;
    // The z step of the running sums, as the reference build executes it (its SASS: FMUL m = cell.z * R.z once, then FFMA v = m * f + v per z):
    // nvcc contracts  v_x += Rcurr_inv.z * cell_size.z * intr.fx  (tsdf_volume.cu:574), so the addend is the EXACT product m * f, not
    // its float rounding.  Adding the rounded product instead differs in the last bit of v_x about once per 10^7 voxel updates, enough
    // to pick the neighbouring depth pixel for a few voxels per frame (found by the 512^3 replay test).
    const float m0z = __fmul_rn(Rcurr_inv.r0.z, cell_size.z), m1z = __fmul_rn(Rcurr_inv.r1.z, cell_size.z);

    float tranc_dist_inv = 1.0f / tranc_dist;

    // ---- conservative frustum interval of this column (not part of the reference; it only removes voxels the
    // exact tests below would reject): with q(z) = q0 + z*dq, q = (fx*p_x, fy*p_y, p_z) in the camera frame, a voxel
    // can be accepted only if p_z > 0 and -0.5 <= u < cols-0.5, -0.5 <= v < rows-0.5.  Margin: 2 voxels + 1 pixel.
    int zlo = z0, zhi = z1;
    {
        const float dqx = Rcurr_inv_0_z_scaled, dqy = Rcurr_inv_1_z_scaled, dqz = Rcurr_inv.r2.z * cell_size.z;
        {   // cheap reject (most threads): every constraint is linear in z, so if both ends of [z0-3, z1+3] violate the same
            // one (with the slack used below) the whole chunk of this column is outside the view frustum
            const float za = (float)(z0 - 3), zb = (float)(z1 + 3);
            const float ax = v_x + za * dqx, ay = v_y + za * dqy, az = v_z + za * dqz;
            const float bx = v_x + zb * dqx, by = v_y + zb * dqy, bz = v_z + zb * dqz;
            const float kx0 = intr.cx + 1.5f, kx1 = intr.cx - cols - 0.5f, ky0 = intr.cy + 1.5f, ky1 = intr.cy - rows - 0.5f;
            const float sl = 2e-3f * (fabsf(v_x) + fabsf(v_y) + (fabsf(v_z) + fabsf(dqz) * V) * (fabsf(kx1) + fabsf(ky1) + fabsf(kx0) + fabsf(ky0)) + (fabsf(dqx) + fabsf(dqy)) * V) + 1e-5f;
            if ((az < -sl && bz < -sl) ||
                (ax + kx0 * az < -sl && bx + kx0 * bz < -sl) || (ax + kx1 * az > sl && bx + kx1 * bz > sl) ||
                (ay + ky0 * az < -sl && by + ky0 * bz < -sl) || (ay + ky1 * az > sl && by + ky1 * bz > sl)) return;
        }
        float lo = -1e30f, hi = 1e30f;
        // each constraint: a + b*z >= 0
        const float ca[5] = { v_z,
                              v_x + (intr.cx + 1.5f) * v_z,
                              -(v_x + (intr.cx - cols - 0.5f) * v_z),
                              v_y + (intr.cy + 1.5f) * v_z,
                              -(v_y + (intr.cy - rows - 0.5f) * v_z) };
        const float cb[5] = { dqz,
                              dqx + (intr.cx + 1.5f) * dqz,
                              -(dqx + (intr.cx - cols - 0.5f) * dqz),
                              dqy + (intr.cy + 1.5f) * dqz,
                              -(dqy + (intr.cy - rows - 0.5f) * dqz) };
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            const float a = ca[c], b = cb[c];
            const float eps = 1e-3f * (fabsf(a) + fabsf(b) * V) + 1e-6f;      // float-rounding slack
            if (fabsf(b) * V <= eps) { if (a < -eps) { lo = 1e30f; hi = -1e30f; } }
            else {
                float zc = -(a + eps) / b;                     // boundary moved outward by eps (either sign of b)
                if (b > 0) lo = fmaxf(lo, zc); else hi = fminf(hi, zc);
            }
        }
        if (lo > hi) return;
        zlo = max(z0, (int)floorf(fmaxf(lo, -4.f)) - 2);
        zhi = min(z1, (int)ceilf(fminf(hi, (float)V + 4.f)) + 3);
        if (zlo >= zhi) return;
    }

    // the running sums at zlo: exactly the bits the reference reaches after zlo steps, in O(binades crossed) instead of O(zlo)
    // dependent FFMAs (kt_replay.cuh; the one-by-one replay was about a quarter of this kernel's issued instructions)
    if (p.seq_replay) {            // KT_INT_SEQ_REPLAY (test hook): the additions one by one, as the reference performs them
        for (int z = 0; z < zlo; ++z) { v_x = __fmaf_rn(m0z, intr.fx, v_x); v_y = __fmaf_rn(m1z, intr.fy, v_y); }
    } else {
        v_x = replay_fma(v_x, m0z, intr.fx, zlo);
        v_y = replay_fma(v_y, m1z, intr.fy, zlo);
    }
    const float* __restrict__ zt = p.ztable;
    const float* __restrict__ depthScaled = p.depth_scaled;
    const float* __restrict__ nmap_curr = p.nmap;
    const uchar3* __restrict__ colors = reinterpret_cast<const uchar3*>(p.rgb);
    const IdxT P = (IdxT)rows * cols;
    const IdxT plane = (IdxT)V * V;
    const IdxT col_off = (IdxT)sy * V + sx;

    // The z loop is processed in batches of ZU voxels in three phases (project + depth gather / sdf test + volume loads /
    // blend + stores) so that ZU independent memory round trips are in flight per thread; the per-voxel arithmetic and the
    // running sums are exactly the reference's (storage addresses of different z never alias, which the compiler cannot know).
    for (int zb = zlo; zb < zhi; zb += ZU) {
        if (MG) {
            // Shared volume: only the storage planes this rank owns are integrated here.  A run of foreign planes is crossed by STEPPING the
            // running sums -- two FFMAs per plane, the reference's own arithmetic -- or, when the run is long (many ranks), by the exact
            // fast-forward; the ownership pattern has period 2^bshift * world, which divides V, so it continues across the cyclic wrap.
            int sz = zb + p.wrap.z; if (sz >= V) sz -= V;
            if (vv_owner(p.vv, sz) != p.vv.rank) {
                const int blk = sz >> p.vv.bshift;
                const int foreign = (p.vv.rank - blk - 1) & (p.vv.world - 1);          // whole foreign blocks between this one and mine
                int skip = (((blk + 1) << p.vv.bshift) - sz) + (foreign << p.vv.bshift);
                skip = min(skip, zhi - zb);
                if (skip <= 48) { for (int k = 0; k < skip; ++k) { v_x = __fmaf_rn(m0z, intr.fx, v_x); v_y = __fmaf_rn(m1z, intr.fy, v_y); } }
                else { v_x = replay_fma(v_x, m0z, intr.fx, skip); v_y = replay_fma(v_y, m1z, intr.fy, skip); }
                zb += skip - ZU;
                continue;
            }
        }
        float vgz[ZU], Dp[ZU];
        IdxT pix[ZU], addr[ZU], caddr[ZU];
        bool ok[ZU];
        float nx[ZU], nz[ZU];
        int16_t tprev[ZU]; uchar4 cprev[ZU]; uchar3 rgbv[ZU]; float4 rgbq[ZU];
#pragma unroll
        for (int u = 0; u < ZU; ++u) {
            const int z = zb + u;
            ok[u] = false;
            if (z < zhi) {
                vgz[u] = zt[z];
                const float z_scaled = zt[V + z];
                float inv_z = 1.0f / __fmaf_rn(Rcurr_inv.r2.z, z_scaled, v_z);             // 1 / (v_z + Rcurr_inv.r2.z * z_scaled)
                if (!(inv_z < 0)) {
                    int2 coo = { __float2int_rn(__fmaf_rn(v_x, inv_z, intr.cx)), __float2int_rn(__fmaf_rn(v_y, inv_z, intr.cy)) };
                    if (coo.x >= 0 && coo.y >= 0 && coo.x < cols && coo.y < rows) {
                        int sz = z + p.wrap.z; if (sz >= V) sz -= V;
                        ok[u] = true;
                        pix[u] = (IdxT)coo.y * cols + coo.x;
                        addr[u] = (IdxT)sz * plane + col_off;
                        caddr[u] = MG ? (IdxT)vv_local_plane(p.vv, sz) * plane + col_off : addr[u];      // colour planes are sharded, local order
                        Dp[u] = depthScaled[pix[u]];
                    }
                }
                v_x = __fmaf_rn(m0z, intr.fx, v_x);
                v_y = __fmaf_rn(m1z, intr.fy, v_y);
            }
        }
        bool upd[ZU], nocol[ZU];
        float tsdf_new[ZU];
#pragma unroll
        for (int u = 0; u < ZU; ++u) {
            upd[u] = false;
            if (ok[u]) {
                float Dp_scaled = Dp[u];
                bool no_color = false;
                if (Dp_scaled < 0.0) { Dp_scaled = -Dp_scaled; no_color = true; }
                float sdf = Dp_scaled - sqrtf(__fmaf_rn(vgz[u], vgz[u], v_g_part_norm));
                if (Dp_scaled != 0 && sdf >= -tranc_dist) {
                    upd[u] = true; nocol[u] = no_color;
                    tsdf_new[u] = fmin(1.0f, sdf * tranc_dist_inv);
                    // (issuing these loads together with the depth gather, before the test, was slower: 78 -> 88 us at 512^3)
                    tprev[u] = p.tsdf[addr[u]];
                    cprev[u] = p.color[caddr[u]];
                    if (PREP) { nx[u] = p.cw[pix[u]]; rgbq[u] = p.rgbf[pix[u]]; }
                    else {
                        nx[u] = nmap_curr[pix[u]];
                        nz[u] = nmap_curr[pix[u] + 2 * P];
                        rgbv[u] = colors[pix[u]];
                    }
                }
            }
        }
#pragma unroll
        for (int u = 0; u < ZU; ++u) {
            if (!upd[u]) continue;
            float tsdf = tsdf_new[u];
            float tsdf_prev = unpack_tsdf(tprev[u]);
            uchar4 c = cprev[u];
            float weight_prev = c.w;
            const float Wrk = 1;
            const short tnew = pack_tsdf(__fmaf_rn(tsdf_prev, weight_prev, tsdf) / (weight_prev + Wrk));   // (F * W + Wrk * tsdf) / (W + Wrk), Wrk = 1
            p.tsdf[addr[u]] = tnew;
            if (MG && !p.mg_no_publish && tnew != tprev[u]) {
                // the owner publishes a changed value to every replica (free-space voxels that stay at 32767 cause no traffic)
                for (int g = 0; g < p.vv.world; ++g) if (g != p.vv.rank) p.vv.tsdf[g][addr[u]] = tnew;
            }
            c.w = min(weight_prev + Wrk, (float)KT_MAX_WEIGHT);
            if (PREP) {
                const float cwv = nx[u];
                if ((__float_as_int(cwv) >= 0 && !nocol[u]) || (c.x == 0 && c.y == 0 && c.z == 0)) {
                    const float Wrkc = fabsf(cwv);
                    const float4 rgb = rgbq[u];
                    float new_x = __fmaf_rn(Wrkc, rgb.x, __fmul_rn(c.x, weight_prev)) / (weight_prev + Wrkc);   // (c * W + Wrkc * rgb) / (W + Wrkc): the reference build fuses Wrkc * rgb into the sum (SASS: FMUL W * c, then FFMA Wrkc * rgb + that)
                    float new_y = __fmaf_rn(Wrkc, rgb.y, __fmul_rn(c.y, weight_prev)) / (weight_prev + Wrkc);
                    float new_z = __fmaf_rn(Wrkc, rgb.z, __fmul_rn(c.z, weight_prev)) / (weight_prev + Wrkc);
                    c.x = sat_u8_rn(new_x);
                    c.y = sat_u8_rn(new_y);
                    c.z = sat_u8_rn(new_z);
                }
            } else {
                float3 ncurr; ncurr.x = nx[u]; ncurr.z = nz[u];
                if (ncurr.z < 0) ncurr.z = -ncurr.z;
                if ((!isnan(ncurr.x) && !nocol[u]) || (c.x == 0 && c.y == 0 && c.z == 0)) {
                    const float Wrkc = (p.angle_color ? min(1.0f, ncurr.z / KT_RGB_VIEW_ANGLE_WEIGHT) : 1.0f) * 2.0f;
                    uchar3 rgb = rgbv[u];
                    float new_x = __fmaf_rn(Wrkc, rgb.x, __fmul_rn(c.x, weight_prev)) / (weight_prev + Wrkc);   // (c * W + Wrkc * rgb) / (W + Wrkc): the reference build fuses Wrkc * rgb into the sum (SASS: FMUL W * c, then FFMA Wrkc * rgb + that)
                    float new_y = __fmaf_rn(Wrkc, rgb.y, __fmul_rn(c.y, weight_prev)) / (weight_prev + Wrkc);
                    float new_z = __fmaf_rn(Wrkc, rgb.z, __fmul_rn(c.z, weight_prev)) / (weight_prev + Wrkc);
                    c.x = min(255, max(0, __float2int_rn(new_x)));
                    c.y = min(255, max(0, __float2int_rn(new_y)));
                    c.z = min(255, max(0, __float2int_rn(new_z)));
                }
            }
            p.color[caddr[u]] = c;
        }
    }
}

int fill_zero(void* p, size_t bytes, cudaStream_t s)
{
    size_t n16 = bytes / 16;
    int grid = (int)((n16 + 255) / 256 < (size_t)device_info().sm_count * 16 ? (n16 + 255) / 256 : (size_t)device_info().sm_count * 16);
    if (grid < 1) grid = 1;
    fill_zero_u4<<<grid, 256, 0, s>>>((uint4*)p, n16);
    KT_LAUNCH_CHECK();
    return 0;
}

// storage index of logical plane 0 for a signed wrap (tsdf_volume.cu:134, :254, :359)
int wrap_base(int current, int V)
{
    int b = current > 0 ? current % V : V - ((-current) % V);
    return b % V;
}

} // namespace

int init_volume(int16_t* tsdf, uint8_t* color, int vol, cudaStream_t s)
{
    size_t n = (size_t)vol * vol * vol;
    int r = fill_zero(tsdf, n * 2, s); if (r) return r;
    return fill_zero(color, n * 4, s);
}

// Semantics of the 12 reference wrappers (SURVEY.md Q13, Appendix B), n = delta - current:
//   forward (n > 0): storage planes base .. base+n   (n+1 planes)
//   back    (n < 0): storage planes base-|n| .. base (|n|+1 planes)
//   X variants only reach round_up_16(|n|) planes from the start of the range (the launch is that wide),
//   which drops the last plane exactly when |n| is a multiple of 16.
int clear_volume(int axis, int back, int16_t* tsdf, uint8_t* color, int vol, int current, int delta, cudaStream_t s)
{
    return clear_volume_shared(axis, back, single_volume(tsdf, color, vol), vol, current, delta, s);
}

int init_shared(const VolumeView& vv, int vol, cudaStream_t s)
{
    const size_t plane = (size_t)vol * vol;
    int r = fill_zero(vv.tsdf[vv.rank], plane * vol * 2, s); if (r) return r;
    return fill_zero(vv.color[vv.rank], plane * (vol / vv.world) * 4, s);
}

int clear_volume_shared(int axis, int back, const VolumeView& vv, int vol, int current, int delta, cudaStream_t s)
{
    const int V = vol;
    const int n = delta - current;
    const int an = n < 0 ? -n : n;
    const int base = wrap_base(current, V);
    int p0 = back ? ((base - an) % V + V) % V : base;
    int count = an + 1;
    if (axis == 0) {
        int reach = (an % 16 != 0) ? (an + 16 - an % 16) : an;
        if (count > reach) count = reach;
    }
    if (count <= 0) return 0;
    if (count > V) count = V;
    int16_t* tsdf = vv.tsdf[vv.rank]; uint8_t* color = vv.color[vv.rank];
    if (axis == 0) {
        size_t total = (size_t)count * V * V;
        int grid = (int)((total + 255) / 256 < (size_t)device_info().sm_count * 16 ? (total + 255) / 256 : (size_t)device_info().sm_count * 16);
        clear_planes_x_kernel<<<grid, 256, 0, s>>>(tsdf, (uchar4*)color, V, p0, count, vv);
    } else {
        size_t total = (size_t)count * V * (V / 8);
        int grid = (int)((total + 255) / 256 < (size_t)device_info().sm_count * 16 ? (total + 255) / 256 : (size_t)device_info().sm_count * 16);
        clear_planes_yz_kernel<<<grid, 256, 0, s>>>(tsdf, color, V, axis, p0, count, vv);
    }
    KT_LAUNCH_CHECK();
    return 0;
}

int color_prep(const float* nmap, const uint8_t* rgb, int rows, int cols, bool angle_color, float* cw, float4* rgbf, cudaStream_t s)
{
    const int n = rows * cols;
    color_prep_kernel<<<div_up(n, 256), 256, 0, s>>>(nmap, reinterpret_cast<const uchar3*>(rgb), n, angle_color, cw, rgbf);
    KT_LAUNCH_CHECK();
    return 0;
}

int integrate(const IntegrateArgs& a, float* ztable_dev, cudaStream_t s)
{
    const int V = a.vol;
    float3 cell = make_float3(a.volume_size.x / V, a.volume_size.y / V, a.volume_size.z / V);   // host division, tsdf_volume.cu:659-661
    static const bool seq_replay = getenv("KT_INT_SEQ_REPLAY") != nullptr;
    ztable_kernel<<<div_up(2 * V, 256), 256, 0, s>>>(ztable_dev, V, cell.z, a.t.z, a.reset_words, a.reset_words ? a.reset_count : 0, a.reset_stride, seq_replay ? 1 : 0);
    KT_LAUNCH_CHECK();
    IntegrateParams p;
    p.depth_scaled = a.depth_scaled; p.rows = a.rows; p.cols = a.cols; p.k = a.k; p.cell = cell; p.Rinv = a.Rinv; p.t = a.t; p.trunc = a.trunc;
    p.tsdf = a.tsdf; p.color = (uchar4*)a.color; p.V = V; p.wrap = wrap_mod3(a.wrap, V); p.rgb = a.rgb; p.nmap = a.nmap_curr; p.angle_color = a.angle_color;
    static int n_chunks = -1, order = -1;          // tuning knobs: KT_INT_ZCHUNKS (default 16), KT_INT_ORDER (0 near-first = default, 1 far-first)
    if (n_chunks < 0) { const char* e = getenv("KT_INT_ZCHUNKS"); n_chunks = e ? atoi(e) : 16; if (n_chunks < 1) n_chunks = 1; }
    if (order < 0) { const char* e = getenv("KT_INT_ORDER"); order = e ? atoi(e) : 0; }
    static int zu = -1;
    if (zu < 0) { const char* e = getenv("KT_INT_ZU"); zu = e ? atoi(e) : 0; }
    static int prep_knob = -1;                      // KT_INT_PREP=0 keeps the per-voxel colour arithmetic (A/B)
    if (prep_knob < 0) { const char* e = getenv("KT_INT_PREP"); prep_knob = e ? atoi(e) : 1; }
    const bool prep = prep_knob != 0 && a.cw && a.rgbf;      // the caller ran color_prep() on this frame's normal map and image
    p.cw = a.cw; p.rgbf = a.rgbf;
    p.ztable = ztable_dev; p.zchunk = V >= 64 ? (V + n_chunks - 1) / n_chunks : V;
    // z chunks: a warp walks its columns' voxels serially, so a chunk's length is the scheduling quantum of the launch; 16 chunks
    // balance that quantum against the per-chunk column setup (KT_INT_ZCHUNKS and tools/stage_ab.py re-measure it).
    p.z_far_first = (a.Rinv.r2.z > 0.f) == (order != 0) ? 1 : 0;          // z component of the camera's viewing axis in the volume frame
    const bool multi = a.multi && a.vv.world > 1;
    p.vv = multi ? a.vv : single_volume(a.tsdf, a.color, V);
    // KT_FORCE_IDX64 (test hook): take the 64-bit index path the 2048^3 volume needs on a volume small enough to check against the reference
    static const bool force64 = getenv("KT_FORCE_IDX64") != nullptr;
    const bool idx32 = !force64 && (size_t)V * V * V <= ((size_t)1 << 31);
    p.lz_lo = 0; p.lz_hi = V;
    p.seq_replay = seq_replay ? 1 : 0;
    static const bool no_publish = getenv("KT_MG_NO_PUBLISH") != nullptr;
    p.mg_no_publish = no_publish ? 1 : 0;
    p.tiles_x = div_up(V, 32); p.tiles_y = div_up(V, 8); p.tile_x0 = 0; p.tile_y0 = 0;
    dim3 block(32, 8), grid(p.tiles_x, p.tiles_y, div_up(V, p.zchunk));
    // Launch only the storage tiles and z chunks the view frustum can reach (kt_frustum.hpp: a conservative box in logical voxel
    // coordinates; the per-column test in the kernel stays).  KT_INT_NOBOX=1 (test hook) launches the whole volume as before.
    static const bool no_box = getenv("KT_INT_NOBOX") != nullptr;
    if (!no_box) {
        const float Rinv9[9] = {a.Rinv.r0.x, a.Rinv.r0.y, a.Rinv.r0.z, a.Rinv.r1.x, a.Rinv.r1.y, a.Rinv.r1.z, a.Rinv.r2.x, a.Rinv.r2.y, a.Rinv.r2.z};
        const float t3[3] = {a.t.x, a.t.y, a.t.z}, k4[4] = {a.k.fx, a.k.fy, a.k.cx, a.k.cy}, cell3[3] = {cell.x, cell.y, cell.z};
        const VoxelBox box = frustum_voxel_box(Rinv9, t3, k4, a.rows, a.cols, V, cell3);
        if (box.empty) return 0;                                       // the camera sees no voxel of the cube: nothing to integrate
        p.lz_lo = box.lo[2]; p.lz_hi = box.hi[2] + 1;
        grid.z = div_up(p.lz_hi - p.lz_lo, p.zchunk);
        if (V % 32 == 0) { int n; cyclic_tile_range(box.lo[0], box.hi[0], p.wrap.x, V, 32, &p.tile_x0, &n); grid.x = n; }
        if (V % 8 == 0) { int n; cyclic_tile_range(box.lo[1], box.hi[1], p.wrap.y, V, 8, &p.tile_y0, &n); grid.y = n; }
    }
    if (multi) {
        if (V & (V - 1)) { set_error("integrate: the shared volume needs a power-of-two resolution"); return -1; }
        // one voxel per step: the walk alternates between owned blocks and stepped-over foreign ones
        if (idx32) { if (prep) integrate_kernel<unsigned int, 1, 6, true, true><<<grid, block, 0, s>>>(p); else integrate_kernel<unsigned int, 1, 6, false, true><<<grid, block, 0, s>>>(p); }
        else { if (prep) integrate_kernel<size_t, 1, 6, true, true><<<grid, block, 0, s>>>(p); else integrate_kernel<size_t, 1, 6, false, true><<<grid, block, 0, s>>>(p); }
    } else if (idx32) {
        // batch depth / CTAs per SM (KT_INT_ZU = 1 or 2 overrides): 2-voxel batches at 4 CTAs/SM while the updated region stays in L2,
        // 1-voxel steps at 6 CTAs/SM from 1024^3, where occupancy hides the HBM latency (tools/stage_ab.py compares them).
        const int variant = zu ? zu : (V >= 1024 ? 1 : 2);
        if (prep && (variant == 1 || variant == 2)) {
            if (variant == 1) integrate_kernel<unsigned int, 1, 6, true><<<grid, block, 0, s>>>(p);
            else integrate_kernel<unsigned int, 2, 4, true><<<grid, block, 0, s>>>(p);
        } else
        if (variant == 1) integrate_kernel<unsigned int, 1, 6><<<grid, block, 0, s>>>(p);
        else integrate_kernel<unsigned int, 2, 4><<<grid, block, 0, s>>>(p);
    }
    else if (prep) integrate_kernel<size_t, 1, 6, true><<<grid, block, 0, s>>>(p);
    else if (zu == 2) integrate_kernel<size_t, 2, 4><<<grid, block, 0, s>>>(p);
    else integrate_kernel<size_t, 1, 6><<<grid, block, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// Cross-GPU barrier over NVLink peer memory (one process per GPU, flag arrays exchanged through CUDA IPC).
namespace {
__global__ void xgpu_barrier_kernel(unsigned int* const* peer_flags, volatile unsigned int* my_flags, int rank, int world, unsigned int epoch, int* error)
{
    const int t = threadIdx.x;
    if (t < world) {
        __threadfence_system();                                  // everything this GPU wrote before (local slab, P2P stores) is visible first
        volatile unsigned int* dst = peer_flags[t] + rank;
        *dst = epoch;
        __threadfence_system();
        const long long t0 = clock64();
        while ((int)(my_flags[t] - epoch) < 0) {
            if (clock64() - t0 > 4000000000LL) { *error = 1 + t; break; }   // ~2 s at 2 GHz: report instead of hanging the GPU
        }
        __threadfence_system();
    }
}
}

int xgpu_barrier(unsigned int* const* peer_flags_dev, unsigned int* my_flags, int rank, int world, unsigned int epoch, int* error_dev, cudaStream_t s)
{
    xgpu_barrier_kernel<<<1, 32, 0, s>>>(peer_flags_dev, my_flags, rank, world, epoch, error_dev);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
