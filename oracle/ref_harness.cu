// TEST INFRASTRUCTURE ONLY (oracle/): never linked into, imported by or executed from the
// product path (kintinuous_b200/).
//
// C-ABI harness around the reference's OWN CUDA operators (src/frontend/cuda/internal.h:299-536),
// compiled by oracle/build_ref.sh from the sources where they lie under the reference checkout (two
// mechanical sed patches for post-Volta warp intrinsics on a temporary copy, VOL made a -D macro;
// SURVEY.md D5/D7). Output: oracle/_ref/libkt_ref_<VOL>.so (git-ignored, travels to the GPU box).
// Nothing from the reference is copied into this repository; this file only CALLS the reference API.
//
// Every buffer crossing this ABI is a raw DEVICE pointer with a compact pitch (cols*sizeof(T)),
// wrapped in the reference's DeviceArray2D(rows, cols, data, step) user-data constructor
// (containers/device_array.hpp:170), so the same buffers can be handed to the product kernels for A/B tests.
#include "internal.h"
#include <cuda_runtime.h>
#include <vector>
#include <cstring>
#include "kt_host_logic.hpp"

typedef unsigned short u16;

template <class T> static DeviceArray2D<T> wrap2(const void* p, int rows, int cols)
{
    return DeviceArray2D<T>(rows, cols, const_cast<void*>(p), (size_t)cols * sizeof(T));
}
static Mat33 toMat33(const float* m) { Mat33 r; std::memcpy(&r, m, 36); return r; }
static float3 toF3(const float* v) { return make_float3(v[0], v[1], v[2]); }

extern "C" {

int ktref_vol() { return VOL; }
int ktref_max_threads() { return MAX_THREADS; }

void ktref_bilateral(const u16* src, u16* dst, int rows, int cols)
{
    DeviceArray2D<u16> s = wrap2<u16>(src, rows, cols), d = wrap2<u16>(dst, rows, cols);
    bilateralFilter(s, d);
    cudaSafeCall(cudaDeviceSynchronize());
}

void ktref_pyrdown(const u16* src, u16* dst, int srows, int scols)
{
    DeviceArray2D<u16> s = wrap2<u16>(src, srows, scols), d = wrap2<u16>(dst, srows / 2, scols / 2);
    pyrDown(s, d);
    cudaSafeCall(cudaDeviceSynchronize());
}

void ktref_vmap(const u16* depth, float* vmap, int rows, int cols, const float* intr)
{
    DeviceArray2D<u16> s = wrap2<u16>(depth, rows, cols);
    DeviceArray2D<float> v = wrap2<float>(vmap, rows * 3, cols);
    createVMap(Intr(intr[0], intr[1], intr[2], intr[3]), s, v);
    cudaSafeCall(cudaDeviceSynchronize());
}

void ktref_nmap(const float* vmap, float* nmap, int rows, int cols)
{
    DeviceArray2D<float> v = wrap2<float>(vmap, rows * 3, cols), n = wrap2<float>(nmap, rows * 3, cols);
    createNMap(v, n);
    cudaSafeCall(cudaDeviceSynchronize());
}

void ktref_transform_maps(const float* vs, const float* ns, const float* R, const float* t, float* vd, float* nd, int rows, int cols)
{
    DeviceArray2D<float> a = wrap2<float>(vs, rows * 3, cols), b = wrap2<float>(ns, rows * 3, cols);
    DeviceArray2D<float> c = wrap2<float>(vd, rows * 3, cols), d = wrap2<float>(nd, rows * 3, cols);
    tranformMaps(a, b, toMat33(R), toF3(t), c, d);
}

void ktref_resize_vmap(const float* in, float* out, int in_rows, int in_cols)
{
    DeviceArray2D<float> a = wrap2<float>(in, in_rows * 3, in_cols), b = wrap2<float>(out, (in_rows / 2) * 3, in_cols / 2);
    resizeVMap(a, b);
}

void ktref_resize_nmap(const float* in, float* out, int in_rows, int in_cols)
{
    DeviceArray2D<float> a = wrap2<float>(in, in_rows * 3, in_cols), b = wrap2<float>(out, (in_rows / 2) * 3, in_cols / 2);
    resizeNMap(a, b);
}

static DeviceArray<JtJJtrSE3>* g_sum = 0;
static DeviceArray<JtJJtrSE3>* g_out = 0;
static DeviceArray<int2>* g_sumRes = 0;
static void ensure_reduce_buffers()
{
    if (!g_sum) {
        g_sum = new DeviceArray<JtJJtrSE3>(); g_sum->create(MAX_THREADS);     // ICPOdometry.cpp:39-40 (Q15)
        g_out = new DeviceArray<JtJJtrSE3>(); g_out->create(1);
        g_sumRes = new DeviceArray<int2>(); g_sumRes->create(MAX_THREADS);    // RGBDOdometry.cpp:45-47
    }
}

// threads/blocks as the reference's callers hard-code them: 128 x 64 (ICPOdometry.cpp:124-125)
void ktref_icp_step(const float* Rcurr, const float* tcurr, const float* vmap_curr, const float* nmap_curr,
                    const float* Rprev_inv, const float* tprev, const float* intr,
                    const float* vmap_g_prev, const float* nmap_g_prev, int rows, int cols,
                    float distThres, float angleThres, float* A_host, float* b_host, float* residual_host)
{
    ensure_reduce_buffers();
    DeviceArray2D<float> vc = wrap2<float>(vmap_curr, rows * 3, cols), nc = wrap2<float>(nmap_curr, rows * 3, cols);
    DeviceArray2D<float> vp = wrap2<float>(vmap_g_prev, rows * 3, cols), np = wrap2<float>(nmap_g_prev, rows * 3, cols);
    icpStep(toMat33(Rcurr), toF3(tcurr), vc, nc, toMat33(Rprev_inv), toF3(tprev), Intr(intr[0], intr[1], intr[2], intr[3]),
            vp, np, distThres, angleThres, *g_sum, *g_out, A_host, b_host, residual_host, 128, 64);
}

static DeviceArray2D<float>* g_depthScaled = 0;

void ktref_integrate(const u16* depth_raw, int rows, int cols, const float* intr, const float* volume_size,
                     const float* Rcurr_inv, const float* tcurr, float trunc, short* tsdf, unsigned char* color,
                     const int* voxelWrap, const unsigned char* rgb, const float* nmap_curr, int angleColor, float* depthScaled)
{
    PtrStepSz<u16> d(rows, cols, const_cast<u16*>(depth_raw), (size_t)cols * 2);
    DeviceArray2D<float> ds = wrap2<float>(depthScaled, rows, cols);
    DeviceArray2D<float> nm = wrap2<float>(nmap_curr, rows * 3, cols);
    PtrStep<short> vol(tsdf, (size_t)VOL * sizeof(short));
    PtrStep<uchar4> cvol((uchar4*)color, (size_t)VOL * sizeof(uchar4));
    PtrStepSz<uchar3> colors(rows, cols, (uchar3*)const_cast<unsigned char*>(rgb), (size_t)cols * 3);
    int3 w = make_int3(voxelWrap[0], voxelWrap[1], voxelWrap[2]);
    integrateTsdfVolume(d, Intr(intr[0], intr[1], intr[2], intr[3]), toF3(volume_size), toMat33(Rcurr_inv), toF3(tcurr), trunc,
                        vol, ds, w, cvol, colors, nm, angleColor != 0);
}

void ktref_raycast(const float* intr, const float* Rcurr, const float* tcurr, float trunc, const float* volume_size,
                   const short* tsdf, float* vmap, float* nmap, int rows, int cols, const int* voxelWrap,
                   unsigned char* vmap_color, const unsigned char* color)
{
    DeviceArray2D<float> v = wrap2<float>(vmap, rows * 3, cols), n = wrap2<float>(nmap, rows * 3, cols);
    DeviceArray2D<uchar4> vc = wrap2<uchar4>(vmap_color, rows, cols);
    PtrStep<short> vol(const_cast<short*>(tsdf), (size_t)VOL * sizeof(short));
    PtrStep<uchar4> cvol((uchar4*)const_cast<unsigned char*>(color), (size_t)VOL * sizeof(uchar4));
    int3 w = make_int3(voxelWrap[0], voxelWrap[1], voxelWrap[2]);
    raycast(Intr(intr[0], intr[1], intr[2], intr[3]), toMat33(Rcurr), toF3(tcurr), trunc, toF3(volume_size), vol, v, n, w, vc, cvol);
    cudaSafeCall(cudaDeviceSynchronize());
}

// GUI taps: generateImage / generateDepth (image_generator.cu:161-230)
void ktref_generate_image(const float* vmap, const float* nmap, const unsigned char* vmap_color, const float* light_pos3, int n_lights,
                          unsigned char* dst_rgb, unsigned char* dst_color_rgb, int rows, int cols)
{
    DeviceArray2D<float> v = wrap2<float>(vmap, rows * 3, cols), n = wrap2<float>(nmap, rows * 3, cols);
    DeviceArray2D<uchar4> vc = wrap2<uchar4>(vmap_color, rows, cols);
    LightSource light; light.number = n_lights; light.pos[0] = make_float3(light_pos3[0], light_pos3[1], light_pos3[2]);
    PtrStepSz<uchar3> d(rows, cols, (uchar3*)dst_rgb, (size_t)cols * 3), dc(rows, cols, (uchar3*)dst_color_rgb, (size_t)cols * 3);
    generateImage(v, n, vc, light, d, dc);
}
void ktref_generate_depth(const float* Rinv, const float* t, const float* vmap, const float* nmap, u16* dst, int rows, int cols, float max_depth)
{
    DeviceArray2D<float> v = wrap2<float>(vmap, rows * 3, cols), n = wrap2<float>(nmap, rows * 3, cols);
    DeviceArray2D<u16> d = wrap2<u16>(dst, rows, cols);
    generateDepth(toMat33(Rinv), toF3(t), v, n, d, max_depth);
    cudaSafeCall(cudaDeviceSynchronize());
}

size_t ktref_extract(const short* tsdf, const float* volume_size, void* out, size_t out_cap, const int* voxelWrap,
                     const unsigned char* color, int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int subsample,
                     const int* realVoxelWrap)
{
    PtrStep<short> vol(const_cast<short*>(tsdf), (size_t)VOL * sizeof(short));
    PtrStep<uchar4> cvol((uchar4*)const_cast<unsigned char*>(color), (size_t)VOL * sizeof(uchar4));
    PtrSz<PointXYZRGB> o((PointXYZRGB*)out, out_cap);
    return extractCloudSlice(vol, toF3(volume_size), o, make_int3(voxelWrap[0], voxelWrap[1], voxelWrap[2]), cvol,
                             minX, maxX, minY, maxY, minZ, maxZ, subsample,
                             make_int3(realVoxelWrap[0], realVoxelWrap[1], realVoxelWrap[2]));
}

void ktref_clear(int axis, int back, short* tsdf, unsigned char* color, int current, int delta)
{
    PtrStep<short> vol(tsdf, (size_t)VOL * sizeof(short));
    PtrStep<uchar4> cvol((uchar4*)color, (size_t)VOL * sizeof(uchar4));
    if (axis == 0 && !back) { clearVolumeX(vol, current, delta); clearVolumeXc(cvol, current, delta); }
    if (axis == 0 && back)  { clearVolumeXBack(vol, current, delta); clearVolumeXBackc(cvol, current, delta); }
    if (axis == 1 && !back) { clearVolumeY(vol, current, delta); clearVolumeYc(cvol, current, delta); }
    if (axis == 1 && back)  { clearVolumeYBack(vol, current, delta); clearVolumeYBackc(cvol, current, delta); }
    if (axis == 2 && !back) { clearVolumeZ(vol, current, delta); clearVolumeZc(cvol, current, delta); }
    if (axis == 2 && back)  { clearVolumeZBack(vol, current, delta); clearVolumeZBackc(cvol, current, delta); }
}

void ktref_init_volume(short* tsdf, unsigned char* color)
{
    PtrStep<short> vol(tsdf, (size_t)VOL * sizeof(short));
    PtrStep<uchar4> cvol((uchar4*)color, (size_t)VOL * sizeof(uchar4));
    initVolume(vol);
    initColorVolume(cvol);
}

// ---- RGB-D odometry operators ----
void ktref_short_depth_to_metres(const u16* src, float* dst, int rows, int cols, int cutOff)
{
    DeviceArray2D<u16> s = wrap2<u16>(src, rows, cols); DeviceArray2D<float> d = wrap2<float>(dst, rows, cols);
    shortDepthToMetres(s, d, cutOff);
    cudaSafeCall(cudaDeviceSynchronize());
}
void ktref_pyrdown_gauss_f(const float* src, float* dst, int srows, int scols)
{
    DeviceArray2D<float> s = wrap2<float>(src, srows, scols), d = wrap2<float>(dst, srows / 2, scols / 2);
    pyrDownGaussF(s, d);
    cudaSafeCall(cudaDeviceSynchronize());
}
void ktref_bgr_to_intensity(const unsigned char* rgb, unsigned char* dst, int rows, int cols)
{
    DeviceArray2D<PixelRGB> s = wrap2<PixelRGB>(rgb, rows, cols); DeviceArray2D<unsigned char> d = wrap2<unsigned char>(dst, rows, cols);
    imageBGRToIntensity(s, d);
    cudaSafeCall(cudaDeviceSynchronize());
}
void ktref_pyrdown_uchar_gauss(const unsigned char* src, unsigned char* dst, int srows, int scols)
{
    DeviceArray2D<unsigned char> s = wrap2<unsigned char>(src, srows, scols), d = wrap2<unsigned char>(dst, srows / 2, scols / 2);
    pyrDownUcharGauss(s, d);
}
void ktref_derivative_images(const unsigned char* src, short* dx, short* dy, int rows, int cols)
{
    DeviceArray2D<unsigned char> s = wrap2<unsigned char>(src, rows, cols);
    DeviceArray2D<short> a = wrap2<short>(dx, rows, cols), b = wrap2<short>(dy, rows, cols);
    computeDerivativeImages(s, a, b);
}
void ktref_project_to_point_cloud(const float* depth, float* cloud, int rows, int cols, const double* intrinsics, int level)
{
    DeviceArray2D<float> d = wrap2<float>(depth, rows, cols);
    DeviceArray2D<float3> c = wrap2<float3>(cloud, rows, cols);
    IntrDoublePrecision k(intrinsics[0], intrinsics[1], intrinsics[2], intrinsics[3]);
    projectToPointCloud(d, c, k, level);
}
void ktref_rgb_residual(float minScale, const short* dIdx, const short* dIdy, const float* lastDepth, const float* nextDepth,
                        const unsigned char* lastImage, const unsigned char* nextImage, void* corresImg, int rows, int cols,
                        float maxDepthDelta, const float* kt, const float* krkinv, int* sigmaSum, int* count)
{
    ensure_reduce_buffers();
    DeviceArray2D<short> a = wrap2<short>(dIdx, rows, cols), b = wrap2<short>(dIdy, rows, cols);
    DeviceArray2D<float> ld = wrap2<float>(lastDepth, rows, cols), nd = wrap2<float>(nextDepth, rows, cols);
    DeviceArray2D<unsigned char> li = wrap2<unsigned char>(lastImage, rows, cols), ni = wrap2<unsigned char>(nextImage, rows, cols);
    DeviceArray2D<DataTerm> ci = wrap2<DataTerm>(corresImg, rows, cols);
    computeRgbResidual(minScale, a, b, ld, nd, li, ni, ci, *g_sumRes, maxDepthDelta, toF3(kt), toMat33(krkinv), *sigmaSum, *count, 128, 256);
}
void ktref_rgb_step(const void* corresImg, float sigma, const float* cloud, float fx, float fy, const short* dIdx, const short* dIdy,
                    float sobelScale, int rows, int cols, float* A_host, float* b_host)
{
    ensure_reduce_buffers();
    DeviceArray2D<DataTerm> ci = wrap2<DataTerm>(corresImg, rows, cols);
    DeviceArray2D<float3> c = wrap2<float3>(cloud, rows, cols);
    DeviceArray2D<short> a = wrap2<short>(dIdx, rows, cols), b = wrap2<short>(dIdy, rows, cols);
    rgbStep(ci, sigma, c, fx, fy, a, b, sobelScale, *g_sum, *g_out, A_host, b_host, 128, 64);
}

} // extern "C"

// ---------------------------------------------------------------------------------------------
// Backend for kto::RefTracker: device memory + the reference operators above.
struct RefCudaBackend {
    void* alloc(size_t bytes) { void* p = 0; cudaSafeCall(cudaMalloc(&p, bytes ? bytes : 1)); return p; }
    void free(void* p) { if (p) cudaFree(p); }
    void zero(void* p, size_t bytes) { cudaSafeCall(cudaMemset(p, 0, bytes)); }
    // blocking copies from/to pageable memory, as DeviceArray2D::upload/download do (device_memory.cpp:258-267)
    void upload(void* dst, const void* src, size_t bytes) { cudaSafeCall(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); }
    void download(void* dst, const void* src, size_t bytes) { cudaSafeCall(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost)); }

    // NOTE: inside the tracker the wrappers are called WITHOUT the extra cudaDeviceSynchronize the
    // standalone ktref_* entry points add, to keep the reference's own sync pattern (SURVEY.md §3.2).
    void bilateral(const u16* s, u16* d, int rows, int cols) { DeviceArray2D<u16> a = wrap2<u16>(s, rows, cols), b = wrap2<u16>(d, rows, cols); bilateralFilter(a, b); }
    void pyrdown(const u16* s, u16* d, int sr, int sc) { DeviceArray2D<u16> a = wrap2<u16>(s, sr, sc), b = wrap2<u16>(d, sr / 2, sc / 2); pyrDown(a, b); }
    void vmap(const u16* depth, float* v, int rows, int cols, kto::IntrF k) { DeviceArray2D<u16> a = wrap2<u16>(depth, rows, cols); DeviceArray2D<float> b = wrap2<float>(v, rows * 3, cols); createVMap(Intr(k.fx, k.fy, k.cx, k.cy), a, b); }
    void nmap(const float* v, float* n, int rows, int cols) { DeviceArray2D<float> a = wrap2<float>(v, rows * 3, cols), b = wrap2<float>(n, rows * 3, cols); createNMap(a, b); }
    void transform_maps(const float* vs, const float* ns, const float* R, const float* t, float* vd, float* nd, int rows, int cols) { ktref_transform_maps(vs, ns, R, t, vd, nd, rows, cols); }
    void resize_vmap(const float* in, float* out, int r, int c) { ktref_resize_vmap(in, out, r, c); }
    void resize_nmap(const float* in, float* out, int r, int c) { ktref_resize_nmap(in, out, r, c); }
    void icp_step(const float* Rc, const float* tc, const float* vc, const float* nc, const float* Rpi, const float* tp, kto::IntrF k,
                  const float* vp, const float* np, int rows, int cols, float dt, float at, float* A, float* b, float* res)
    { float in[4] = {k.fx, k.fy, k.cx, k.cy}; ktref_icp_step(Rc, tc, vc, nc, Rpi, tp, in, vp, np, rows, cols, dt, at, A, b, res); }
    void integrate(const u16* depth, int rows, int cols, kto::IntrF k, const float* vs, const float* Rinv, const float* t, float trunc,
                   short* tsdf, unsigned char* color, int vol, const int* wrap, const unsigned char* rgb, const float* nm, int angleColor, float* ds)
    { (void)vol; float in[4] = {k.fx, k.fy, k.cx, k.cy}; ktref_integrate(depth, rows, cols, in, vs, Rinv, t, trunc, tsdf, color, wrap, rgb, nm, angleColor, ds); }
    void raycast(kto::IntrF k, const float* R, const float* t, float trunc, const float* vs, const short* tsdf, int vol, float* v, float* n,
                 int rows, int cols, const int* wrap, unsigned char* vc, const unsigned char* color)
    {
        (void)vol;
        DeviceArray2D<float> a = wrap2<float>(v, rows * 3, cols), b = wrap2<float>(n, rows * 3, cols);
        DeviceArray2D<uchar4> c = wrap2<uchar4>(vc, rows, cols);
        PtrStep<short> volp(const_cast<short*>(tsdf), (size_t)VOL * sizeof(short));
        PtrStep<uchar4> cvol((uchar4*)const_cast<unsigned char*>(color), (size_t)VOL * sizeof(uchar4));
        ::raycast(Intr(k.fx, k.fy, k.cx, k.cy), toMat33(R), toF3(t), trunc, toF3(vs), volp, a, b, make_int3(wrap[0], wrap[1], wrap[2]), c, cvol);
    }
    size_t extract(const short* tsdf, const float* vs, int vol, void* out, size_t cap, const int* wrap, const unsigned char* color,
                   int x0, int x1, int y0, int y1, int z0, int z1, int sub, const int* realWrap)
    { (void)vol; return ktref_extract(tsdf, vs, out, cap, wrap, color, x0, x1, y0, y1, z0, z1, sub, realWrap); }
    void clear(int axis, int back, short* tsdf, unsigned char* color, int vol, int cur, int delta) { (void)vol; ktref_clear(axis, back, tsdf, color, cur, delta); }
    void init_volume(short* tsdf, unsigned char* color, int vol) { (void)vol; ktref_init_volume(tsdf, color); }
    void short_depth_to_metres(const u16* s, float* d, int rows, int cols, int cut) { DeviceArray2D<u16> a = wrap2<u16>(s, rows, cols); DeviceArray2D<float> b = wrap2<float>(d, rows, cols); shortDepthToMetres(a, b, cut); }
    void pyrdown_gauss_f(const float* s, float* d, int sr, int sc) { DeviceArray2D<float> a = wrap2<float>(s, sr, sc), b = wrap2<float>(d, sr / 2, sc / 2); pyrDownGaussF(a, b); }
    void bgr_to_intensity(const unsigned char* s, unsigned char* d, int rows, int cols) { DeviceArray2D<PixelRGB> a = wrap2<PixelRGB>(s, rows, cols); DeviceArray2D<unsigned char> b = wrap2<unsigned char>(d, rows, cols); imageBGRToIntensity(a, b); }
    void pyrdown_uchar_gauss(const unsigned char* s, unsigned char* d, int sr, int sc) { ktref_pyrdown_uchar_gauss(s, d, sr, sc); }
    void derivative_images(const unsigned char* s, short* dx, short* dy, int rows, int cols) { ktref_derivative_images(s, dx, dy, rows, cols); }
    void project_to_point_cloud(const float* depth, float* cloud, int rows, int cols, kto::IntrD k, int level)
    { double in[4] = {k.fx, k.fy, k.cx, k.cy}; ktref_project_to_point_cloud(depth, cloud, rows, cols, in, level); }
    void rgb_residual(float minScale, const short* dx, const short* dy, const float* ld, const float* nd, const unsigned char* li,
                      const unsigned char* ni, void* ci, int rows, int cols, float mdd, const float* kt, const float* krk, int* sigma, int* count)
    { ktref_rgb_residual(minScale, dx, dy, ld, nd, li, ni, ci, rows, cols, mdd, kt, krk, sigma, count); }
    void rgb_step(const void* ci, float sigma, const float* cloud, float fx, float fy, const short* dx, const short* dy, float ss,
                  int rows, int cols, float* A, float* b)
    { ktref_rgb_step(ci, sigma, cloud, fx, fy, dx, dy, ss, rows, cols, A, b); }
};

static RefCudaBackend g_backend;
#define KT_TRK_TYPE kto::RefTracker<RefCudaBackend>
#define KT_BACKEND g_backend
#define KT_FN(name) ktref_tracker_##name
#include "kt_tracker_cabi.inc"
