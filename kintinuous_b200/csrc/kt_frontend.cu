// kintinuous_b200 -- the fused per-frame front end: everything between "a depth / colour frame arrived" and "the odometry can start"
// in TWO launches (the reference: 12 for ICP-only, 24 + 6 device allocations / frees for the photometric modes).
//
// Replaces (reference, src/frontend/cuda/), as ONE pipeline instead of one kernel + one cudaDeviceSynchronize per function:
//   launch 1  bilateral_scale_kernel (kt_pyramid.cu)   bilateralFilter (bilateral_pyrdown.cu:60-99) + scaleDepth (tsdf_volume.cu:491-538)
//   launch 2  frontend_pyramid_kernel (this file)      pyrDown x3 (bilateral_pyrdown.cu:102-136), createVMap / createNMap x4 (maps.cu:57-155),
//             the per-pixel half of the colour integration (tsdf_volume.cu:601-622) and, for -r / -ri, populateRGBDData +
//             computeDerivativeImages: shortDepthToMetres, imageBGRToIntensity, pyrDownGaussF x3, pyrDownUcharGauss x3, the 3x3
//             gradient at all four levels (bilateral_pyrdown.cu:172-331, RGBDOdometry.cpp:140-175)
//
// Design:  A CTA owns a 64 x 32 pixel tile of level 0 and produces ITS part of every output of every pyramid level from shared
// memory: the tile is staged once with the halo the three 5x5 decimations need (level l computes its owned pixels plus a halo of
// HL_l / HR_l pixels, HL_l = 2 HL_{l+1} + 2, HR_l = 2 HR_{l+1} + 1: 14 / 15 pixels at level 0 for the depth pyramid, 22 / 15 with the
// photometric pyramids whose gradient needs one more left neighbour at level 3).  The halo is recomputed by the neighbouring CTAs --
// 2.4x redundant work on the cheap 25-tap decimations (the 169-tap bilateral filter is NOT recomputed: it is launch 1) -- which buys
// independence: no level ever goes back to HBM before the next one reads it, the vertex map is never re-read to make normals, and
// 150 CTAs (about one wave on 132 SMs) replace 11-23 dependent launches of <= 76 800 threads.  Per-pixel arithmetic is the
// reference's, expression by expression (window clipping Q1, integer weight count Q2, stale y/z planes Q7, the gradient's tap walk),
// with the contractions its build has (read off the SASS: fma(g, .587, fma(r, .114, b * .299)), fma(v, w, sum)) written out.
// Bound: HBM streaming of the outputs (51 B per level-0 pixel ICP-only, 74 B with the photometric set), latency of three
// dependent in-CTA levels.
#include "kt_ops.h"
#include "kt_frontend.cuh"

namespace kt {

namespace {

enum { FE_TW = 64, FE_TH = 32, FE_THREADS = 512 };

// geometry of the computed region per level (in that level's pixels): owned tile + HL pixels left / top + HR pixels right / bottom
template <bool RGBD, int L> struct FeL {
    enum { HL = 2 * FeL<RGBD, L + 1>::HL + 2, HR = 2 * FeL<RGBD, L + 1>::HR + 1, W = (FE_TW >> L) + HL + HR, H = (FE_TH >> L) + HL + HR, N = W * H };
};
template <bool RGBD> struct FeL<RGBD, 3> { enum { HL = RGBD ? 1 : 0, HR = 1, W = (FE_TW >> 3) + HL + HR, H = (FE_TH >> 3) + HL + HR, N = W * H }; };
template <bool RGBD> struct FeGeom {
    enum { N_ALL = FeL<RGBD, 0>::N + FeL<RGBD, 1>::N + FeL<RGBD, 2>::N + FeL<RGBD, 3>::N, SMEM = N_ALL * (2 + (RGBD ? 5 : 0)) + 64 };
};

struct FrontendParams {
    const uint16_t* depth_f; const uint16_t* depth_raw; const uchar3* rgb;
    int rows, cols;
    uint16_t* depths[LEVELS];
    float* vmaps[LEVELS]; float* nmaps[LEVELS]; const float* vstale[LEVELS]; const float* nstale[LEVELS];
    float fx_inv[LEVELS], fy_inv[LEVELS], cx[LEVELS], cy[LEVELS];
    float* cw; float4* rgbf; int angle_color;
    int cut_off; float* depth_m[LEVELS]; uint8_t* intensity[LEVELS]; int16_t* dIdx[LEVELS]; int16_t* dIdy[LEVELS];
};

#define KT_RGB_VIEW_ANGLE_WEIGHT 0.75f

// a level's shared-memory tile addressed in that level's GLOBAL pixel coordinates
template <class T> struct Tile {
    const T* base; int x0, y0, pitch;                       // (x0, y0): global coordinate of element 0
    __device__ __forceinline__ T operator()(int y, int x) const { return base[(y - y0) * pitch + (x - x0)]; }
};

struct FeSmem { float* sf[LEVELS]; uint16_t* sd[LEVELS]; uint8_t* si[LEVELS]; };

// one pyramid level of the CTA: (L > 0) compute the level's region from the level below in shared memory, then write every output of
// the pixels the CTA owns at this level
template <bool RGBD, int L>
__device__ __forceinline__ void fe_level(const FrontendParams& p, const FeSmem& sm, int X0, int Y0)
{
    typedef FeL<RGBD, L> G;
    const int tid = threadIdx.x;
    const int lrows = p.rows >> L, lcols = p.cols >> L;
    const int XL = X0 >> L, YL = Y0 >> L;
    const int gx0 = XL - G::HL, gy0 = YL - G::HL;
    if (L > 0) {
        enum { LS = L > 0 ? L - 1 : 0 };
        typedef FeL<RGBD, LS> GS;
        const int srows = p.rows >> LS, scols = p.cols >> LS;
        const Tile<uint16_t> td = {sm.sd[LS], (X0 >> LS) - GS::HL, (Y0 >> LS) - GS::HL, GS::W};
        const Tile<float> tf = {sm.sf[LS], td.x0, td.y0, GS::W};
        const Tile<uint8_t> ti = {sm.si[LS], td.x0, td.y0, GS::W};
        for (int i = tid; i < G::N; i += FE_THREADS) {
            const int ly = i / G::W, lx = i - ly * G::W;
            const int gx = gx0 + lx, gy = gy0 + ly;
            if (gx < 0 || gy < 0 || gx >= lcols || gy >= lrows) { sm.sd[L][i] = 0; if (RGBD) { sm.sf[L][i] = 0.f; sm.si[L][i] = 0; } continue; }
            if (p.depth_f) sm.sd[L][i] = pyrdown_depth_px(td, gx, gy, srows, scols);
            if (RGBD) { sm.sf[L][i] = pyrdown_float_px(tf, gx, gy, srows, scols); sm.si[L][i] = pyrdown_uchar_px(ti, gx, gy, srows, scols); }
        }
        __syncthreads();
    }
    const Tile<uint16_t> td = {sm.sd[L], gx0, gy0, G::W};
    const Tile<float> tf = {sm.sf[L], gx0, gy0, G::W};
    const Tile<uint8_t> ti = {sm.si[L], gx0, gy0, G::W};
    const int ow = FE_TW >> L, oh = FE_TH >> L;
    const size_t P = (size_t)lrows * lcols;
    const float fx_inv = p.fx_inv[L], fy_inv = p.fy_inv[L], cx = p.cx[L], cy = p.cy[L];
    float* __restrict__ vm = p.vmaps[L]; float* __restrict__ nm = p.nmaps[L];
    const float* __restrict__ vst = p.vstale[L]; const float* __restrict__ nst = p.nstale[L];
    const float nan = qnan();
    for (int i = tid; i < ow * oh; i += FE_THREADS) {
        const int oy = i / ow, ox = i - oy * ow;
        const int u = XL + ox, v = YL + oy;
        if (u >= lcols || v >= lrows) continue;
        const size_t gi = (size_t)v * lcols + u;
        if (vm) {
            const int d00 = td(v, u);
            if (L > 0) p.depths[L][gi] = (uint16_t)d00;
            // computeVmapKernel + computeNmapKernel (maps.cu:57-120); Q7: an invalid pixel gets NaN in its x plane only -- its y / z planes
            // keep what they held (the previous frame's values: vst / nst when the outputs are a spare buffer set)
            float3 v00;
            const bool ok00 = vertex_of(d00, u, v, fx_inv, fy_inv, cx, cy, v00);
            if (ok00) { vm[gi] = v00.x; vm[gi + P] = v00.y; vm[gi + 2 * P] = v00.z; }
            else { vm[gi] = nan; if (vst) { vm[gi + P] = vst[gi + P]; vm[gi + 2 * P] = vst[gi + 2 * P]; } }
            bool okn = false;
            float nx_seen = nan, nz_seen = 0.f;            // what a later reader of the normal map finds at this pixel (x and z planes)
            if (ok00 && u != lcols - 1 && v != lrows - 1) {
                float3 v01, v10;
                const bool ok01 = vertex_of(td(v, u + 1), u + 1, v, fx_inv, fy_inv, cx, cy, v01);
                const bool ok10 = vertex_of(td(v + 1, u), u, v + 1, fx_inv, fy_inv, cx, cy, v10);
                if (ok01 && ok10) {
                    const float3 n = normalized3(cross3(diff3(v01, v00), diff3(v10, v00)));
                    nm[gi] = n.x; nm[gi + P] = n.y; nm[gi + 2 * P] = n.z;
                    okn = true; nx_seen = n.x; nz_seen = n.z;
                }
            }
            if (!okn) {
                nm[gi] = nan;
                if (nst) { const float sy = nst[gi + P], sz = nst[gi + 2 * P]; nm[gi + P] = sy; nm[gi + 2 * P] = sz; nz_seen = sz; }
                else if (L == 0 && p.cw) nz_seen = nm[gi + 2 * P];
            }
            if (L == 0 && p.cw) {
                // per-pixel half of the colour update (tsdf_volume.cu:601-622): view-angle weight, its sign carries isnan(n_x); RGB as float
                float nz = nz_seen;
                if (nz < 0) nz = -nz;
                const float Wrkc = (p.angle_color ? min(1.0f, nz / KT_RGB_VIEW_ANGLE_WEIGHT) : 1.0f) * 2.0f;
                p.cw[gi] = isnan(nx_seen) ? -Wrkc : Wrkc;
                const uchar3 c = p.rgb[gi];
                p.rgbf[gi] = make_float4((float)c.x, (float)c.y, (float)c.z, 0.f);
            }
        }
        if (RGBD) {
            p.depth_m[L][gi] = tf(v, u);
            p.intensity[L][gi] = ti(v, u);
            int16_t gx, gy;
            gradient_px(ti, u, v, lrows, lcols, gx, gy);
            p.dIdx[L][gi] = gx; p.dIdy[L][gi] = gy;
        }
    }
}

template <bool RGBD>
__global__ void __launch_bounds__(FE_THREADS)
frontend_pyramid_kernel(const FrontendParams p)
{
    extern __shared__ __align__(16) unsigned char fe_smem[];
    const int tid = threadIdx.x;
    FeSmem sm;
    {   // carve: floats first (alignment), then u16, then u8
        const int n[LEVELS] = {FeL<RGBD, 0>::N, FeL<RGBD, 1>::N, FeL<RGBD, 2>::N, FeL<RGBD, 3>::N};
        unsigned char* q = fe_smem;
        for (int l = 0; l < LEVELS; ++l) { sm.sf[l] = (float*)q; if (RGBD) q += (size_t)n[l] * 4; }
        for (int l = 0; l < LEVELS; ++l) { sm.sd[l] = (uint16_t*)q; q += (size_t)n[l] * 2; }
        for (int l = 0; l < LEVELS; ++l) { sm.si[l] = (uint8_t*)q; if (RGBD) q += (size_t)n[l]; }
    }
    const int X0 = blockIdx.x * FE_TW, Y0 = blockIdx.y * FE_TH;
    const int rows = p.rows, cols = p.cols;
    // ---- stage level 0 (filtered depth; raw depth in metres and intensity for the photometric set) ----
    {
        typedef FeL<RGBD, 0> G;
        const int gx0 = X0 - G::HL, gy0 = Y0 - G::HL;
        for (int i = tid; i < G::N; i += FE_THREADS) {
            const int ly = i / G::W, lx = i - ly * G::W;
            const int gx = gx0 + lx, gy = gy0 + ly;
            const bool in = gx >= 0 && gx < cols && gy >= 0 && gy < rows;
            const size_t gi = (size_t)gy * cols + gx;
            sm.sd[0][i] = (in && p.depth_f) ? p.depth_f[gi] : (uint16_t)0;
            if (RGBD) {
                const int raw = in ? (int)p.depth_raw[gi] : 0;
                sm.sf[0][i] = depth_to_metres(raw, p.cut_off);
                sm.si[0][i] = in ? rgb_to_intensity(p.rgb[gi]) : (uint8_t)0;
            }
        }
    }
    __syncthreads();
    fe_level<RGBD, 0>(p, sm, X0, Y0);
    fe_level<RGBD, 1>(p, sm, X0, Y0);
    fe_level<RGBD, 2>(p, sm, X0, Y0);
    fe_level<RGBD, 3>(p, sm, X0, Y0);
}

} // namespace

int frontend_pyramid(const FrontendArgs& a, cudaStream_t s)
{
    FrontendParams p;
    p.depth_f = a.depth_f; p.depth_raw = a.depth_raw; p.rgb = reinterpret_cast<const uchar3*>(a.rgb);
    p.rows = a.rows; p.cols = a.cols;
    for (int l = 0; l < LEVELS; ++l) {
        const Intr kl = intr_level(a.k, l);
        p.depths[l] = a.depths[l]; p.vmaps[l] = a.vmaps ? a.vmaps[l] : 0; p.nmaps[l] = a.nmaps ? a.nmaps[l] : 0;
        p.vstale[l] = a.vstale ? a.vstale[l] : 0; p.nstale[l] = a.nstale ? a.nstale[l] : 0;
        p.fx_inv[l] = 1.f / kl.fx; p.fy_inv[l] = 1.f / kl.fy; p.cx[l] = kl.cx; p.cy[l] = kl.cy;      // 1/fx on the HOST, maps.cu:135
        p.depth_m[l] = a.depth_m ? a.depth_m[l] : 0; p.intensity[l] = a.intensity ? a.intensity[l] : 0;
        p.dIdx[l] = a.dIdx ? a.dIdx[l] : 0; p.dIdy[l] = a.dIdy ? a.dIdy[l] : 0;
    }
    p.cw = a.cw; p.rgbf = a.rgbf; p.angle_color = a.angle_color ? 1 : 0; p.cut_off = a.cut_off;
    const bool rgbd = a.depth_m != 0;
    DeviceInfo& di = device_info();
    if (!(di.configured & 4u)) {
        cudaFuncSetAttribute((const void*)frontend_pyramid_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FeGeom<true>::SMEM);
        cudaFuncSetAttribute((const void*)frontend_pyramid_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FeGeom<false>::SMEM);
        di.configured |= 4u;
    }
    dim3 grid(div_up(a.cols, FE_TW), div_up(a.rows, FE_TH));
    if (rgbd) frontend_pyramid_kernel<true><<<grid, FE_THREADS, FeGeom<true>::SMEM, s>>>(p);
    else frontend_pyramid_kernel<false><<<grid, FE_THREADS, FeGeom<false>::SMEM, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
