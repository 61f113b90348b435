// kintinuous_b200 -- depth pyramid and vertex / normal maps (sm_90a).
//
// Replaces (reference file:line, src/frontend/cuda/):
//   bilateralFilter / bilateralKernel      bilateral_pyrdown.cu:60-99, :333-343
//   pyrDown / pyrDownGaussKernel           bilateral_pyrdown.cu:102-136, :345-354
//   createVMap / computeVmapKernel         maps.cu:57-80, :123-138
//   createNMap / computeNmapKernel         maps.cu:83-121, :140-155
//   tranformMaps / tranformMapsKernel      maps.cu:157-222
//   resizeVMap/NMap / resizeMapKernel      maps.cu:225-308
// Design: the bilateral filter stages a (4+12)x(32+12) depth tile (as float) in shared memory once per
// CTA (169 taps/pixel come from smem, not L1); vertex and normal maps of ALL pyramid levels are
// produced by ONE launch straight from the depth pyramid (the vertex map is never re-read to make
// normals); per-pixel arithmetic keeps the reference's expression order (see kt_common.cuh).
// Roofline: HBM-bound streaming except the bilateral filter, which is instruction-issue / MUFU(ex2)-bound
// (169 __expf per pixel, 9 instructions per tap); algorithmic bytes: DESIGN.md section 4.
#include "kt_ops.h"
#include "kt_frontend.cuh"

namespace kt {

namespace {

const float SIGMA_COLOR = 30.f;      // mm   (bilateral_pyrdown.cu:56)
const float SIGMA_SPACE = 4.5f;      // px   (bilateral_pyrdown.cu:57)

// 32x4-pixel CTAs: 640x480 is not a whole number of waves of 2048 threads per SM, and with 512-thread CTAs the last few of 600 run
// alone after everyone else; 128-thread CTAs make that tail one small CTA long.
enum { BIL_TX = 32, BIL_TY = 4, BIL_R = 6, BIL_W = BIL_TX + 2 * BIL_R, BIL_H = BIL_TY + 2 * BIL_R };

// One pixel's 13x13 window from the float tile, taps in the reference's order (rows, then columns).  PRED: window clipped to
// [dx_lo, dx_hi) x [dy_lo, dy_hi) (image borders, Q1); otherwise the full window, everything known at compile time.
// The depth tile is held as float so that a tap needs ONE special-function-unit op (ex2) instead of three: the reference's
// (float)tmp and (float)((value - tmp)^2) int->float conversions run on the same 16-lane unit as ex2 and were the bound.
// Exactness: depths < 2^16 are exact in float, so is their difference; RN(diff * diff) equals the int->float conversion of the
// exact integer square as long as the square does not overflow int32 (|diff| <= 46340, checked per CTA by the caller).
template <bool PRED>
__device__ __forceinline__ float bilateral_window(const float (*tile)[BIL_W + 1], int ly, int lx, float value, float ks, float kc,
                                                  int dx_lo, int dx_hi, int dy_lo, int dy_hi)
{
    float sum1 = 0, sum2 = 0;
    // clipped taps contribute weight * 0: fma(tmp, 0, sum1) == sum1 and sum2 + 0 == sum2 exactly, so masking is bit-identical to
    // skipping them and keeps the unrolled window free of branches
    float mx[2 * BIL_R + 1];
    if (PRED) {
#pragma unroll
        for (int dx = -BIL_R; dx <= BIL_R; ++dx) mx[dx + BIL_R] = (dx >= dx_lo && dx < dx_hi) ? 1.f : 0.f;
    }
#pragma unroll
    for (int dy = -BIL_R; dy <= BIL_R; ++dy) {
        const float* trow = tile[ly + BIL_R + dy];
        const float my = (!PRED || (dy >= dy_lo && dy < dy_hi)) ? 1.f : 0.f;
#pragma unroll
        for (int dx = -BIL_R; dx <= BIL_R; ++dx) {
            const float tmp = trow[lx + BIL_R + dx];
            const float space2 = (float)(dx * dx + dy * dy);
            const float diff = __fsub_rn(value, tmp);
            const float color2 = __fmul_rn(diff, diff);
            // the contraction the reference's loop compiles to (checked in SASS): fma(space2, k_s, color2 * k_c)
            const float e = __fmaf_rn(space2, ks, __fmul_rn(color2, kc));
            float weight = __expf(-e);
            if (PRED) weight = __fmul_rn(weight, __fmul_rn(mx[dx + BIL_R], my));
            sum1 = __fmaf_rn(tmp, weight, sum1);
            sum2 = __fadd_rn(sum2, weight);
        }
    }
    return sum1 / sum2;
}

// scaleDepth (tsdf_volume.cu:491-538) for the pixel at tile position (ly, lx): the depth along the ray, D * |((x - cx) / fx, (y - cy) / fy, 1)| / 1000,
// negated ("do not fuse colour here") when more than 5 pixels of its 7x7 window -- clipped like every window of the reference, exclusive and
// to cols-1 / rows-1 (Q1) -- differ by more than 200 mm or the pixel itself is empty.  Depths and their differences are exact in float.
__device__ __forceinline__ float scale_depth_px(const float (*tile)[BIL_W + 1], int ly, int lx, int x, int y, int rows, int cols, const Intr& intr, bool angleColor)
{
    const float Df = tile[ly + BIL_R][lx + BIL_R];
    const int Dp = (int)Df;
    const float xl = (x - intr.cx) / intr.fx;
    const float yl = (y - intr.cy) / intr.fy;
    const float lambda = sqrtf(__fadd_rn(__fmaf_rn(xl, xl, __fmul_rn(yl, yl)), 1.f));     // sqrtf(xl * xl + yl * yl + 1), contraction pinned
    if (angleColor) {
        const int dx_lo = max(-3, -x), dx_hi = min(4, cols - 1 - x), dy_lo = max(-3, -y), dy_hi = min(4, rows - 1 - y);
        int count = 0;
        if (Dp == 0) count = max(0, dx_hi - dx_lo) * max(0, dy_hi - dy_lo);
        else {
#pragma unroll
            for (int dy = -3; dy <= 3; ++dy)
#pragma unroll
                for (int dx = -3; dx <= 3; ++dx)
                    if (dy >= dy_lo && dy < dy_hi && dx >= dx_lo && dx < dx_hi && fabsf(Df - tile[ly + BIL_R + dy][lx + BIL_R + dx]) > 200.f) ++count;
        }
        if (count > 5) return -Dp * lambda / 1000.f;
    }
    return Dp * lambda / 1000.f;
}

// bilateralFilter and scaleDepth share the raw-depth tile: one launch produces the filtered depth (dst) and / or the ray-scaled depth
// for the integration (scaled).
template <bool BIL, bool SCALE>
__global__ void __launch_bounds__(BIL_TX * BIL_TY)
bilateral_scale_kernel(const uint16_t* __restrict__ src, uint16_t* __restrict__ dst, float* __restrict__ scaled, int rows, int cols,
                       float sigma_space2_inv_half, float sigma_color2_inv_half, const Intr intr, bool angleColor)
{
    __shared__ float tile[BIL_H][BIL_W + 1];
    const int x0 = blockIdx.x * BIL_TX, y0 = blockIdx.y * BIL_TY;
    int big = 0;
    for (int i = threadIdx.y * BIL_TX + threadIdx.x; i < BIL_H * BIL_W; i += BIL_TX * BIL_TY) {
        int ty = i / BIL_W, tx = i - ty * BIL_W;
        int gx = x0 + tx - BIL_R, gy = y0 + ty - BIL_R;
        const int v = (gx >= 0 && gx < cols && gy >= 0 && gy < rows) ? (int)src[(size_t)gy * cols + gx] : 0;
        tile[ty][tx] = (float)v;
        big |= (v > 46340);
    }
    const int any_big = __syncthreads_or(big);
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= cols || y >= rows) return;
    if (SCALE) scaled[(size_t)y * cols + x] = scale_depth_px(tile, threadIdx.y, threadIdx.x, x, y, rows, cols, intr, angleColor);
    if (!BIL) return;

    const int D = BIL_R * 2 + 1;
    const float value_f = tile[threadIdx.y + BIL_R][threadIdx.x + BIL_R];
    if (!any_big) {
        float q;
        if (x0 >= BIL_R && y0 >= BIL_R && x0 + BIL_TX - 1 + BIL_R + 1 <= cols - 1 && y0 + BIL_TY - 1 + BIL_R + 1 <= rows - 1)
            q = bilateral_window<false>(tile, threadIdx.y, threadIdx.x, value_f, sigma_space2_inv_half, sigma_color2_inv_half, 0, 0, 0, 0);
        else   // window [max(x-6,0), min(x+7, cols-1)) x [max(y-6,0), min(y+7, rows-1)), exclusive and clipped to cols-1 / rows-1: Q1
            q = bilateral_window<true>(tile, threadIdx.y, threadIdx.x, value_f, sigma_space2_inv_half, sigma_color2_inv_half,
                                       max(-BIL_R, -x), min(BIL_R + 1, cols - 1 - x), max(-BIL_R, -y), min(BIL_R + 1, rows - 1 - y));
        int res = __float2int_rn(q);
        dst[(size_t)y * cols + x] = (uint16_t)max(0, min(res, 32767));
        return;
    }
    // a depth above 46 340 mm in the tile: (value - tmp)^2 overflows int32 in the reference; this CTA reproduces its integer arithmetic,
    // overflow included, on the same tile
    const int value = (int)value_f;
    float sum1 = 0, sum2 = 0;
    const int cy0 = max(y - D / 2, 0), cy1 = min(y - D / 2 + D, rows - 1), cx0 = max(x - D / 2, 0), cx1 = min(x - D / 2 + D, cols - 1);
    for (int cy = cy0; cy < cy1; ++cy) {
        const float* trow = tile[cy - y0 + BIL_R];
        for (int cx = cx0; cx < cx1; ++cx) {
            const int tmp = (int)trow[cx - x0 + BIL_R];
            const float space2 = (x - cx) * (x - cx) + (y - cy) * (y - cy);
            const float color2 = (value - tmp) * (value - tmp);
            const float weight = __expf(-(space2 * sigma_space2_inv_half + color2 * sigma_color2_inv_half));
            sum1 += tmp * weight;
            sum2 += weight;
        }
    }
    int res = __float2int_rn(sum1 / sum2);
    dst[(size_t)y * cols + x] = (uint16_t)max(0, min(res, 32767));
}

// pyrDown (bilateral_pyrdown.cu:102-136, :345-354) at operator level: one thread per output pixel around pyrdown_depth_px
// (kt_frontend.cuh), the function the tracker's fused front end evaluates on shared-memory tiles.
__global__ void __launch_bounds__(256)
pyrdown_gauss_kernel(const uint16_t* __restrict__ src, uint16_t* __restrict__ dst, int srows, int scols, int drows, int dcols)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dcols || y >= drows) return;
    const GlobalSrc<uint16_t> s = {src, scols};
    dst[(size_t)y * dcols + x] = pyrdown_depth_px(s, x, y, srows, scols);
}

__device__ __forceinline__ bool vertex_from_depth(const uint16_t* __restrict__ depth, int cols, int u, int v,
                                                  float fx_inv, float fy_inv, float cx, float cy, float3& out)
{
    float z = depth[(size_t)v * cols + u] / 1000.f;        // mm -> m
    if (z != 0) {
        out.x = __fmul_rn(__fmul_rn(z, (u - cx)), fx_inv);        // rounded products: never fused with the normal's differences (kt_frontend.cuh)
        out.y = __fmul_rn(__fmul_rn(z, (v - cy)), fy_inv);
        out.z = z;
        return true;
    }
    return false;
}

__global__ void __launch_bounds__(256)
vmap_kernel(const uint16_t* __restrict__ depth, float* __restrict__ vmap, int rows, int cols, float fx_inv, float fy_inv, float cx, float cy)
{
    int u = threadIdx.x + blockIdx.x * blockDim.x;
    int v = threadIdx.y + blockIdx.y * blockDim.y;
    if (u >= cols || v >= rows) return;
    float3 p;
    size_t P = (size_t)rows * cols, i = (size_t)v * cols + u;
    if (vertex_from_depth(depth, cols, u, v, fx_inv, fy_inv, cx, cy, p)) { vmap[i] = p.x; vmap[i + P] = p.y; vmap[i + 2 * P] = p.z; }
    else vmap[i] = qnan();                                 // Q7: only the x plane is invalidated
}

__global__ void __launch_bounds__(256)
nmap_kernel(const float* __restrict__ vmap, float* __restrict__ nmap, int rows, int cols)
{
    int u = threadIdx.x + blockIdx.x * blockDim.x;
    int v = threadIdx.y + blockIdx.y * blockDim.y;
    if (u >= cols || v >= rows) return;
    size_t P = (size_t)rows * cols, i = (size_t)v * cols + u;
    if (u == cols - 1 || v == rows - 1) { nmap[i] = qnan(); return; }
    float3 v00, v01, v10;
    v00.x = vmap[i]; v01.x = vmap[i + 1]; v10.x = vmap[i + cols];
    if (!isnan(v00.x) && !isnan(v01.x) && !isnan(v10.x)) {
        v00.y = vmap[i + P]; v01.y = vmap[i + 1 + P]; v10.y = vmap[i + cols + P];
        v00.z = vmap[i + 2 * P]; v01.z = vmap[i + 1 + 2 * P]; v10.z = vmap[i + cols + 2 * P];
        float3 r = normalized3(cross3(diff3(v01, v00), diff3(v10, v00)));
        nmap[i] = r.x; nmap[i + P] = r.y; nmap[i + 2 * P] = r.z;
    } else nmap[i] = qnan();
}

struct MapsParams { MapsLevel lv[LEVELS]; };

// All levels in one launch: blockIdx.z = level, grid sized for level 0.
__global__ void __launch_bounds__(256)
maps_pyramid_kernel(const MapsParams p)
{
    const MapsLevel& L = p.lv[blockIdx.z];
    const int rows = L.rows, cols = L.cols;
    int u = threadIdx.x + blockIdx.x * blockDim.x;
    int v = threadIdx.y + blockIdx.y * blockDim.y;
    if (u >= cols || v >= rows) return;
    const float fx_inv = L.fx_inv, fy_inv = L.fy_inv, cx = L.k.cx, cy = L.k.cy;   // 1/fx is computed on the HOST (maps.cu:135)
    const size_t P = (size_t)rows * cols, i = (size_t)v * cols + u;
    const float nan = qnan();
    float3 v00;
    bool ok00 = vertex_from_depth(L.depth, cols, u, v, fx_inv, fy_inv, cx, cy, v00);
    float* vm = L.vmap; float* nm = L.nmap;
    // Q7: like the reference, an invalid pixel only gets NaN in its x plane; the y/z planes keep what
    // they held (the integrate kernel can read a stale n_z for colour weighting, tsdf_volume.cu:601-622,
    // so reproducing the staleness keeps colour parity with the reference over a sequence).
    // When the maps are built ahead of time into a spare buffer set, 'what they held' is the previous frame's map (vstale / nstale).
    if (ok00) { vm[i] = v00.x; vm[i + P] = v00.y; vm[i + 2 * P] = v00.z; }
    else { vm[i] = nan; if (L.vstale) { vm[i + P] = L.vstale[i + P]; vm[i + 2 * P] = L.vstale[i + 2 * P]; } }
    bool okn = false;
    if (ok00 && u != cols - 1 && v != rows - 1) {
        float3 v01, v10;
        bool ok01 = vertex_from_depth(L.depth, cols, u + 1, v, fx_inv, fy_inv, cx, cy, v01);
        bool ok10 = vertex_from_depth(L.depth, cols, u, v + 1, fx_inv, fy_inv, cx, cy, v10);
        if (ok01 && ok10) {
            float3 n = normalized3(cross3(diff3(v01, v00), diff3(v10, v00)));
            nm[i] = n.x; nm[i + P] = n.y; nm[i + 2 * P] = n.z;
            okn = true;
        }
    }
    if (!okn) { nm[i] = nan; if (L.nstale) { nm[i + P] = L.nstale[i + P]; nm[i + 2 * P] = L.nstale[i + 2 * P]; } }
}

struct TransformParams { TransformLevel lv[LEVELS]; Mat33 R; float3 t; };

__global__ void __launch_bounds__(256)
transform_maps_kernel(const TransformParams p)
{
    const TransformLevel& L = p.lv[blockIdx.z];
    const int rows = L.rows, cols = L.cols;
    int x = threadIdx.x + blockIdx.x * blockDim.x;
    int y = threadIdx.y + blockIdx.y * blockDim.y;
    if (x >= cols || y >= rows) return;
    const float nan = qnan();
    const size_t P = (size_t)rows * cols, i = (size_t)y * cols + x;
    float3 vsrc, vdst = make_float3(nan, nan, nan);
    vsrc.x = L.vs[i];
    if (!isnan(vsrc.x)) {
        vsrc.y = L.vs[i + P]; vsrc.z = L.vs[i + 2 * P];
        vdst = add3(mul33(p.R, vsrc), p.t);
        L.vd[i + P] = vdst.y; L.vd[i + 2 * P] = vdst.z;
    }
    L.vd[i] = vdst.x;
    float3 nsrc, ndst = make_float3(nan, nan, nan);
    nsrc.x = L.ns[i];
    if (!isnan(nsrc.x)) {
        nsrc.y = L.ns[i + P]; nsrc.z = L.ns[i + 2 * P];
        ndst = mul33(p.R, nsrc);
        L.nd[i + P] = ndst.y; L.nd[i + 2 * P] = ndst.z;
    }
    L.nd[i] = ndst.x;
}

template <bool normalize>
__global__ void __launch_bounds__(256)
resize_map_kernel(int drows, int dcols, int srows, int scols, const float* __restrict__ input, float* __restrict__ output)
{
    int x = threadIdx.x + blockIdx.x * blockDim.x;
    int y = threadIdx.y + blockIdx.y * blockDim.y;
    if (x >= dcols || y >= drows) return;
    const float nan = qnan();
    const size_t SP = (size_t)srows * scols, DP = (size_t)drows * dcols;
    const size_t s = (size_t)(2 * y) * scols + 2 * x, d = (size_t)y * dcols + x;
    float x00 = input[s], x01 = input[s + 1], x10 = input[s + scols], x11 = input[s + scols + 1];
    if (isnan(x00) || isnan(x01) || isnan(x10) || isnan(x11)) {
        output[d] = nan;
        return;
    }
    float3 n;
    n.x = (x00 + x01 + x10 + x11) / 4;
    n.y = (input[s + SP] + input[s + SP + 1] + input[s + SP + scols] + input[s + SP + scols + 1]) / 4;
    n.z = (input[s + 2 * SP] + input[s + 2 * SP + 1] + input[s + 2 * SP + scols] + input[s + 2 * SP + scols + 1]) / 4;
    if (normalize) n = normalized3(n);
    output[d] = n.x; output[d + DP] = n.y; output[d + 2 * DP] = n.z;
}

} // namespace

int bilateral_scale(const uint16_t* src, uint16_t* dst, float* scaled, int rows, int cols, const Intr& k, bool angle_color, cudaStream_t s)
{
    dim3 block(BIL_TX, BIL_TY), grid(div_up(cols, BIL_TX), div_up(rows, BIL_TY));
    const float ks = 0.5f / (SIGMA_SPACE * SIGMA_SPACE), kc = 0.5f / (SIGMA_COLOR * SIGMA_COLOR);
    if (dst && scaled) bilateral_scale_kernel<true, true><<<grid, block, 0, s>>>(src, dst, scaled, rows, cols, ks, kc, k, angle_color);
    else if (dst) bilateral_scale_kernel<true, false><<<grid, block, 0, s>>>(src, dst, scaled, rows, cols, ks, kc, k, angle_color);
    else if (scaled) bilateral_scale_kernel<false, true><<<grid, block, 0, s>>>(src, dst, scaled, rows, cols, ks, kc, k, angle_color);
    else return 0;
    KT_LAUNCH_CHECK();
    return 0;
}

int bilateral(const uint16_t* src, uint16_t* dst, int rows, int cols, cudaStream_t s)
{
    Intr k = {1.f, 1.f, 0.f, 0.f};
    return bilateral_scale(src, dst, 0, rows, cols, k, false, s);
}

int scale_depth(const uint16_t* depth, float* scaled, int rows, int cols, const Intr& k, bool angle_color, cudaStream_t s)
{
    return bilateral_scale(depth, 0, scaled, rows, cols, k, angle_color, s);
}

int pyrdown(const uint16_t* src, uint16_t* dst, int srows, int scols, cudaStream_t s)
{
    int drows = srows / 2, dcols = scols / 2;
    dim3 block(32, 8), grid(div_up(dcols, 32), div_up(drows, 8));
    pyrdown_gauss_kernel<<<grid, block, 0, s>>>(src, dst, srows, scols, drows, dcols);
    KT_LAUNCH_CHECK();
    return 0;
}

int create_vmap(const Intr& k, const uint16_t* depth, float* vmap, int rows, int cols, cudaStream_t s)
{
    dim3 block(32, 8), grid(div_up(cols, 32), div_up(rows, 8));
    vmap_kernel<<<grid, block, 0, s>>>(depth, vmap, rows, cols, 1.f / k.fx, 1.f / k.fy, k.cx, k.cy);
    KT_LAUNCH_CHECK();
    return 0;
}

int create_nmap(const float* vmap, float* nmap, int rows, int cols, cudaStream_t s)
{
    dim3 block(32, 8), grid(div_up(cols, 32), div_up(rows, 8));
    nmap_kernel<<<grid, block, 0, s>>>(vmap, nmap, rows, cols);
    KT_LAUNCH_CHECK();
    return 0;
}

int create_maps_pyramid(const MapsLevel* levels, int n, cudaStream_t s)
{
    MapsParams p = {};
    for (int i = 0; i < n; ++i) { p.lv[i] = levels[i]; p.lv[i].fx_inv = 1.f / levels[i].k.fx; p.lv[i].fy_inv = 1.f / levels[i].k.fy; }
    for (int i = n; i < LEVELS; ++i) p.lv[i] = p.lv[n - 1];
    dim3 block(32, 8), grid(div_up(levels[0].cols, 32), div_up(levels[0].rows, 8), n);
    maps_pyramid_kernel<<<grid, block, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

int transform_maps_pyramid(const TransformLevel* levels, int n, const Mat33& R, const float3& t, cudaStream_t s)
{
    TransformParams p;
    for (int i = 0; i < n; ++i) p.lv[i] = levels[i];
    for (int i = n; i < LEVELS; ++i) p.lv[i] = levels[n - 1];
    p.R = R; p.t = t;
    dim3 block(32, 8), grid(div_up(levels[0].cols, 32), div_up(levels[0].rows, 8), n);
    transform_maps_kernel<<<grid, block, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

int transform_maps(const float* vs, const float* ns, const Mat33& R, const float3& t, float* vd, float* nd, int rows, int cols, cudaStream_t s)
{
    TransformLevel L = {vs, ns, vd, nd, rows, cols};
    return transform_maps_pyramid(&L, 1, R, t, s);
}

int resize_map(const float* in, float* out, int in_rows, int in_cols, bool normalize, cudaStream_t s)
{
    int drows = in_rows / 2, dcols = in_cols / 2;
    dim3 block(32, 8), grid(div_up(dcols, 32), div_up(drows, 8));
    if (normalize) resize_map_kernel<true><<<grid, block, 0, s>>>(drows, dcols, in_rows, in_cols, in, out);
    else resize_map_kernel<false><<<grid, block, 0, s>>>(drows, dcols, in_rows, in_cols, in, out);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
