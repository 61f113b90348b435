// kintinuous_b200 -- photometric RGB-D odometry: pre-processing, per-pixel correspondence / residual,
// Jacobian row and the 6x6 reduction (optionally merged with the ICP normal equations, "-ri").
//
// Replaces (reference, src/frontend/):
//   shortDepthToMetres / short2FloatKernel              cuda/bilateral_pyrdown.cu:235-245, :404-411
//   imageBGRToIntensity / bgr2IntensityKernel           cuda/bilateral_pyrdown.cu:247-259, :413-420
//   pyrDownGaussF / pyrDownKernelGaussF                 cuda/bilateral_pyrdown.cu:201-233, :356-378
//   pyrDownUcharGauss / pyrDownKernelIntensityGauss     cuda/bilateral_pyrdown.cu:172-199, :380-402
//   computeDerivativeImages / applyKernel               cuda/bilateral_pyrdown.cu:271-331
//   projectToPointCloud / projectPointsKernel           cuda/maps.cu:311-345
//   computeRgbResidual / RGBResidual / residualKernel   cuda/reduce.cu:668-864
//   rgbStep / RGBReduction / rgbKernel                  cuda/reduce.cu:423-607
//   host half of RGBDOdometry::getIncrementalTransformation   RGBDOdometry.cpp:205-370
// Design: no per-call device allocation or free (the reference allocates the 25-tap table and the reduce
// scratch on every call, SURVEY.md section 3.2); the warp (K R K^-1, K t) of each iteration is rebuilt on the
// device from the running estimate; the sigma of the robust weight and the Gauss-Newton solve live in the
// reduction tails, so an iteration is 2 launches (3 with ICP) and no host round trip.  The tracker itself uses rgbd_frame_kernel:
// the whole coarse-to-fine loop of -r / -ri in ONE cooperative launch (two grid barriers per iteration: count / sigma, then the sums),
// correspondences kept in registers between the residual pass and the Jacobian pass.
#include "kt_ops.h"
#include "kt_solve.cuh"
#include "kt_reduce.cuh"
#include "kt_frame.cuh"
#include "kt_frontend.cuh"

namespace kt {

namespace {

// Operator-level pre-processing kernels (kt_op_short_depth_to_metres / _bgr_to_intensity / _pyrdown_gauss_f / _pyrdown_uchar_gauss /
// _derivative_images / _project_to_point_cloud): one thread per output pixel around the per-pixel functions of kt_frontend.cuh -- the
// same functions the tracker's fused front end evaluates on shared-memory tiles (tests/test_gpu_ops.py holds the two bit-identical).
enum PreOp { PRE_METRES, PRE_INTENSITY, PRE_DOWN_F, PRE_DOWN_U8, PRE_GRADIENT };
struct PreParams { const void* src; void* dst; void* dst2; int rows, cols, srows, scols, cut_off; };

template <int OP>
__global__ void __launch_bounds__(256)
preprocess_kernel(const PreParams p)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= p.cols || y >= p.rows) return;
    const size_t i = (size_t)y * p.cols + x;
    if (OP == PRE_METRES) ((float*)p.dst)[i] = depth_to_metres((int)((const uint16_t*)p.src)[i], p.cut_off);
    else if (OP == PRE_INTENSITY) ((uint8_t*)p.dst)[i] = rgb_to_intensity(((const uchar3*)p.src)[i]);
    else if (OP == PRE_DOWN_F) { const GlobalSrc<float> s = {(const float*)p.src, p.scols}; ((float*)p.dst)[i] = pyrdown_float_px(s, x, y, p.srows, p.scols); }
    else if (OP == PRE_DOWN_U8) { const GlobalSrc<uint8_t> s = {(const uint8_t*)p.src, p.scols}; ((uint8_t*)p.dst)[i] = pyrdown_uchar_px(s, x, y, p.srows, p.scols); }
    else {
        const GlobalSrc<uint8_t> s = {(const uint8_t*)p.src, p.cols};
        int16_t gx, gy;
        gradient_px(s, x, y, p.rows, p.cols, gx, gy);
        ((int16_t*)p.dst)[i] = gx; ((int16_t*)p.dst2)[i] = gy;
    }
}

// projectToPointCloud (maps.cu:311-345): last-frame depth -> float3 point, intrinsics in double
__global__ void __launch_bounds__(256)
project_points_kernel(const float* __restrict__ depth, float3* __restrict__ cloud, int rows, int cols,
                      const double invFx, const double invFy, const double cx, const double cy)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= cols || y >= rows) return;
    const size_t i = (size_t)y * cols + x;
    const float z = depth[i];
    cloud[i] = make_float3((float)((x - cx) * z * invFx), (float)((y - cy) * z * invFy), z);
}

// 16-byte correspondence record, byte-compatible with the reference's DataTerm (cuda/internal.h:90-96)
struct DataTerm { short2 zero; short2 one; float diff; bool valid; };

struct ResidualParams { RgbLevelArgs a; OdomState* st; int* partials; };

// (K R K^-1, K t) from the inverse of the running estimate (RGBDOdometry.cpp:209-231), double then float.
__device__ inline void build_warp(const double* T, double fx, double fy, double cx, double cy, float* krkinv, float* kt)
{
    double R[9], t[3];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R[i * 3 + j] = T[j * 4 + i];          // R^T
    for (int i = 0; i < 3; ++i) t[i] = -(R[i * 3 + 0] * T[3] + R[i * 3 + 1] * T[7] + R[i * 3 + 2] * T[11]);
    const double K[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1};
    const double Ki[9] = {1.0 / fx, 0, -cx / fx, 0, 1.0 / fy, -cy / fy, 0, 0, 1};
    double KR[9];
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) { double s = 0; for (int k = 0; k < 3; ++k) s += K[a * 3 + k] * R[k * 3 + b]; KR[a * 3 + b] = s; }
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) { double s = 0; for (int k = 0; k < 3; ++k) s += KR[a * 3 + k] * Ki[k * 3 + b]; krkinv[a * 3 + b] = (float)s; }
    for (int a = 0; a < 3; ++a) { double s = 0; for (int k = 0; k < 3; ++k) s += K[a * 3 + k] * t[k]; kt[a] = (float)s; }
}

// Pose-independent half of a photometric correspondence (reduce.cu:709-733): the 4x4 neighbourhood of the next image, the gradient
// magnitude and the next depth of pixel idx.  Returns 0 for a pixel that cannot correspond, else 1 | I_next << 8, with its gradient in gr
// and its depth in d1.
__device__ __forceinline__ unsigned int rgb_precheck(const RgbLevelArgs& a, int idx, short2& gr, float& d1)
{
    const int cols = a.cols, rows = a.rows;
    const int i = idx / cols, j0 = idx - i * cols;
    if (!(j0 < cols - 5 && i < rows - 1)) return 0;
    bool valid = true;
    for (int u = max(i - 2, 0); u < min(i + 2, rows); u++)
        for (int v = max(j0 - 2, 0); v < min(j0 + 2, cols); v++)
            valid = valid && (a.next_image[(size_t)u * cols + v] > 0);
    if (!valid) return 0;
    gr.x = a.dIdx[idx]; gr.y = a.dIdy[idx];
    float mTwo = (gr.x * gr.x) + (gr.y * gr.y);
    if (!(mTwo >= a.min_scale)) return 0;
    d1 = a.next_depth[idx];
    if (isnan(d1)) return 0;
    return 1u | ((unsigned int)a.next_image[idx] << 8);
}

// Per-iteration half (reduce.cu:735-764): warp pixel (x, y) at next depth d1 into the last frame with (K R K^-1, K t) and test the last
// frame's depth and intensity there.  True for a correspondence, with its last-frame pixel (u0, v0), depth d0 and diff = I_next - I_last.
__device__ __forceinline__ bool rgb_correspond(const Mat33& krkinv, const float3& kt, int x, int y, float d1, unsigned int i_next,
                                               const float* __restrict__ lastDepth, const uint8_t* __restrict__ lastImage, int cols, int rows,
                                               float maxDepthDelta, int& u0, int& v0, float& d0, float& diff)
{
    float transformed_d1 = (float)(d1 * (krkinv.r2.x * x + krkinv.r2.y * y + krkinv.r2.z) + kt.z);
    u0 = __float2int_rn((d1 * (krkinv.r0.x * x + krkinv.r0.y * y + krkinv.r0.z) + kt.x) / transformed_d1);
    v0 = __float2int_rn((d1 * (krkinv.r1.x * x + krkinv.r1.y * y + krkinv.r1.z) + kt.y) / transformed_d1);
    if (!(u0 >= 0 && v0 >= 0 && u0 < cols && v0 < rows)) return false;
    d0 = __ldg(&lastDepth[(size_t)v0 * cols + u0]);
    const unsigned int il = __ldg(&lastImage[(size_t)v0 * cols + u0]);
    if (!(d0 > 0 && fabsf(transformed_d1 - d0) <= maxDepthDelta && il != 0)) return false;
    diff = static_cast<float>(i_next) - static_cast<float>(il);
    return true;
}

// One Jacobian row of RGBReduction (reduce.cu:443-480), added to sum: robust weight 1/(sigma + |diff|) (1 when sigma == -1), the next
// image's gradient (gx, gy) and the last frame's point.
template <int S>
__device__ __forceinline__ void rgb_pixel_row(float sigma, float diff, short gx, short gy, const float3& cloudPoint, float sobelScale, float fx, float fy,
                                              float (&sum)[S])
{
    float w = sigma + fabsf(diff);
    w = w > 1.19209290E-07F ? 1.0f / w : 1.0f;
    if (sigma == -1) w = 1;
    float row[7];
    row[6] = -w * diff;
    float invz = 1.0 / cloudPoint.z;
    float dI_dx_val = w * sobelScale * gx;
    float dI_dy_val = w * sobelScale * gy;
    float v0 = dI_dx_val * fx * invz;
    float v1 = dI_dy_val * fy * invz;
    float v2 = -(v0 * cloudPoint.x + v1 * cloudPoint.y) * invz;
    row[0] = v0; row[1] = v1; row[2] = v2;
    row[3] = -cloudPoint.z * v1 + cloudPoint.y * v2;
    row[4] = cloudPoint.z * v0 - cloudPoint.x * v2;
    row[5] = -cloudPoint.y * v0 + cloudPoint.x * v1;
    accumulate_row(sum, row);
}

__global__ void __launch_bounds__(RED_THREADS)
residual_kernel(const ResidualParams p, int use_state_warp)
{
    __shared__ float s_w[12];
    __shared__ int s_cnt[RED_THREADS / 32][2];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
    if (tid == 0) {
        if (use_state_warp) build_warp(p.st->resultRt, p.a.Kfx, p.a.Kfy, p.a.Kcx, p.a.Kcy, s_w, s_w + 9);
        else { for (int k = 0; k < 9; ++k) s_w[k] = p.st->krkinv[k]; for (int k = 0; k < 3; ++k) s_w[9 + k] = p.st->kt[k]; }
    }
    __syncthreads();
    const Mat33 krkinv = mat33_rows(s_w);
    const float3 kt = make_float3(s_w[9], s_w[10], s_w[11]);
    const int cols = p.a.cols, rows = p.a.rows, N = cols * rows;
    DataTerm* __restrict__ corresImg = (DataTerm*)p.a.corres;

    int2 sum = {0, 0};
    for (int k = blockIdx.x * RED_THREADS + tid; k < N; k += gridDim.x * RED_THREADS) {
        const int y = k / cols, x = k - y * cols;
        int2 value = {0, 0};
        DataTerm corres;
        corres.zero = make_short2(0, 0); corres.one = make_short2(0, 0); corres.diff = 0.f;
        corres.valid = false;
        short2 gr; float d1; int u0, v0; float d0, diff;
        const unsigned int meta = rgb_precheck(p.a, k, gr, d1);
        if (meta && rgb_correspond(krkinv, kt, x, y, d1, meta >> 8, p.a.last_depth, p.a.last_image, cols, rows, p.a.max_depth_delta, u0, v0, d0, diff)) {
            corres.zero.x = u0; corres.zero.y = v0;
            corres.one.x = x; corres.one.y = y;
            corres.diff = diff;
            corres.valid = true;
            value.x = 1;
            value.y = diff * diff;           // Q5: truncated to int per pixel
        }
        corresImg[k] = corres;
        sum.x += value.x;
        sum.y += value.y;
    }
    // integer reduction (order-independent): shuffle -> smem -> one partial per CTA -> last CTA totals
    for (int o = 16; o > 0; o >>= 1) { sum.x += __shfl_down_sync(0xffffffffu, sum.x, o); sum.y += __shfl_down_sync(0xffffffffu, sum.y, o); }
    if ((tid & 31) == 0) { s_cnt[tid >> 5][0] = sum.x; s_cnt[tid >> 5][1] = sum.y; }
    __syncthreads();
    if (tid == 0) {
        int a = 0, b = 0;
        for (int w = 0; w < RED_THREADS / 32; ++w) { a += s_cnt[w][0]; b += s_cnt[w][1]; }
        p.partials[blockIdx.x * 2] = a; p.partials[blockIdx.x * 2 + 1] = b;
        __threadfence();
        unsigned int ticket = atomicInc(&p.st->blocks_done_rgb, gridDim.x - 1);
        s_last = (ticket == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid == 0) {
        int a = 0, b = 0;
        for (int g = 0; g < (int)gridDim.x; ++g) { a += __ldcg(&p.partials[g * 2]); b += __ldcg(&p.partials[g * 2 + 1]); }
        p.st->rgb_count = a;
        p.st->rgb_sigma = b;
    }
}

struct RgbStepParams { RgbLevelArgs a; OdomState* st; float* partials; float* trace; int mode; float sigma_override; };

__global__ void __launch_bounds__(RED_THREADS)
rgb_step_kernel(const RgbStepParams p)
{
    __shared__ float s_red[RED_THREADS / 32][32];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
    // Q3: sigmaVal = sqrt((float)sigma / rgbSize == 0 ? 1 : rgbSize)  (RGBDOdometry.cpp:253) -- computed like the host does
    float sigma;
    if (p.mode == 0) sigma = p.sigma_override;
    else {
        const int sg = p.st->rgb_sigma, cnt = p.st->rgb_count;
        sigma = (float)sqrt((double)(((float)sg / cnt == 0) ? 1 : cnt));
    }
    const int cols = p.a.cols, rows = p.a.rows, N = cols * rows;
    const DataTerm* __restrict__ corresImg = (const DataTerm*)p.a.corres;
    const float3* __restrict__ cloud = (const float3*)p.a.cloud;
    const int16_t* __restrict__ dIdx = p.a.dIdx; const int16_t* __restrict__ dIdy = p.a.dIdy;

    float sum[NSUM];
#pragma unroll
    for (int k = 0; k < NSUM; ++k) sum[k] = 0.f;
    for (int i = blockIdx.x * RED_THREADS + tid; i < N; i += gridDim.x * RED_THREADS) {
        const DataTerm corresp = corresImg[i];
        if (!corresp.valid) continue;
        const float3 cloudPoint = cloud[(size_t)corresp.zero.y * cols + corresp.zero.x];
        const size_t g = (size_t)corresp.one.y * cols + corresp.one.x;
        rgb_pixel_row(sigma, corresp.diff, dIdx[g], dIdy[g], cloudPoint, p.a.sobel_scale, p.a.fx, p.a.fy, sum);
    }
    if (!grid_reduce29(sum, p.partials, &p.st->blocks_done, s_red, &s_last)) return;

    if (tid < NSUM) p.st->sums_rgb[tid] = s_red[0][tid];
    if (tid == 0) {
        OdomState* st = p.st;
        float A[36], b[6];
        unpack_normal_equations(s_red[0], A, b);
        if (p.trace) {
            float* t = p.trace + (size_t)st->iter * TRACE_STRIDE;
            for (int k = 0; k < 36; ++k) t[k] = A[k];
            for (int k = 0; k < 6; ++k) t[36 + k] = b[k];
            t[42] = (float)st->rgb_sigma; t[43] = (float)st->rgb_count;
        }
        if (p.mode != 0) {
            double dA[36], db[6];
            if (p.mode == 2) {                                  // RGBDOdometry.cpp:316-321
                float Ai[36], bi[6];
                unpack_normal_equations(st->sums_icp, Ai, bi);
                const double w = 10;
                for (int k = 0; k < 36; ++k) dA[k] = (double)A[k] + w * w * (double)Ai[k];
                for (int k = 0; k < 6; ++k) db[k] = (double)b[k] + w * (double)bi[k];
            } else {
                for (int k = 0; k < 36; ++k) dA[k] = A[k];
                for (int k = 0; k < 6; ++k) db[k] = b[k];
            }
            gauss_newton_update(dA, db, st);
            st->iter += 1;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Whole-frame RGB-D odometry (-r) and combined ICP + RGB-D (-ri): all levels and iterations in ONE cooperative launch,
// the photometric twin of icp_frame_kernel (kt_icp.cu).  Per level, once: the pose-independent part of the residual test
// (4x4 neighbourhood of the next image, gradient magnitude, depth validity: reduce.cu:709-733) and the pixel's depth /
// gradients / intensity are staged per thread in shared memory.  Per iteration:
//   pass A  correspondence + photometric residual per pixel (reduce.cu:735-764), kept in REGISTERS for pass B (the
//           reference writes and re-reads a 16-byte DataTerm image); with -ri the point-to-plane sums of the same
//           pixels are accumulated in the same pass;          -> grid barrier 1: count, sigma^2 (+ 29 ICP sums)
//   pass B  Jacobian rows with the robust weight 1/(sigma + |diff|) (reduce.cu:443-480); the last-frame point is
//           rebuilt from its depth (maps.cu:311-329 arithmetic) instead of reading a float3 cloud
//                                                               -> grid barrier 2: 29 sums, FP64 solve in every CTA.
struct RgbdFrameParams {
    IcpLevelArgs icp[LEVELS];
    RgbLevelArgs rgb[LEVELS];
    int iters[LEVELS];
    float pose12[12];
    OdomState* st;
    unsigned long long* xwords;    // exchange words (kt_frame.cuh, XW_WORDS), zero at launch
    float* trace;
    int* timeout;
    float* host_pose; unsigned int host_seq;      // optional mapped host record: pose (12), time-out (1), sequence number (1)
    int stage_k;               // chunks of FRAME_THREADS pixels per CTA (<= RGBD_MAX_K)
    int with_icp;
};

enum { RGBD_MAX_K = 5 };

template <bool WITH_ICP>
__global__ void __launch_bounds__(FRAME_THREADS, 1)
rgbd_frame_kernel(const RgbdFrameParams p)
{
    extern __shared__ __align__(128) float s_dyn[];
    // dynamic smem: [ICP stage: 6 x K x 512 floats (WITH_ICP)] [d1: K x 512 floats] [grad: K x 512 x short2] [meta: K x 512 x uint]
    __shared__ FramePose s_pose;
    __shared__ float s_w[12];
    __shared__ float s_red[FRAME_THREADS / 32][32];
    __shared__ double s_sumd[32];          // merged normal equations in double, written by the lanes that own the components
    __shared__ int s_cnt[FRAME_THREADS / 32][2];
    __shared__ int s_tot[2];
    __shared__ __align__(8) unsigned long long s_mbar;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int G = gridDim.x, K = p.stage_k;
    float* s_stage = s_dyn;
    float* s_d1 = s_dyn + (WITH_ICP ? (size_t)6 * K * FRAME_THREADS : 0);
    short2* s_grad = reinterpret_cast<short2*>(s_d1 + (size_t)K * FRAME_THREADS);
    unsigned int* s_meta = reinterpret_cast<unsigned int*>(s_grad + (size_t)K * FRAME_THREADS);       // bit 0: precheck, bits 8..15: I_next

    Mat33 Rprev_inv; float3 tprev;
    frame_begin(s_pose, p.pose12, &s_mbar, Rprev_inv, tprev);

    int it = 0, ex = 0;                      // iteration / exchange counters (two exchanges per iteration)
    GridSumState gs; gs.prev[0] = 0ull; gs.prev[1] = 0ull;
    GridSumState gs_lo = gs;                 // low words of exchange 2 (grid_sum_words_wide)
    // where lane l's component of the photometric sums lands in a trace record; slots 42 / 43 hold sigma and count instead
    int trace_a = -1, trace_b = -1;
    if (lane < 27) trace_slots(lane, trace_a, trace_b);
    double icp_total = 0.0;                  // warp 0, lane l: grid total of ICP component l of this iteration
    unsigned int stage_parity = 0;
    for (int level = LEVELS - 1; level >= 0; --level) {
        if (p.iters[level] == 0) continue;
        const RgbLevelArgs& a = p.rgb[level];
        const int cols = a.cols, rows = a.rows, N = cols * rows;
        const int n_chunks = (N + G * FRAME_THREADS - 1) / (G * FRAME_THREADS);
        const float* __restrict__ lastDepth = a.last_depth;
        const uint8_t* __restrict__ lastImage = a.last_image;
        const float maxDepthDelta = a.max_depth_delta, fx = a.fx, fy = a.fy, sobelScale = a.sobel_scale;
        const double invFx = 1.0f / a.Kfx, invFy = 1.0f / a.Kfy, dcx = a.Kcx, dcy = a.Kcy;      // projectToPointCloud (maps.cu:342)
        // ---- per-level staging ----
        __syncthreads();
        if (WITH_ICP && tid == 0) {
            const IcpLevelArgs& ia = p.icp[level];
            unsigned int total = 0;
            for (int k = 0; k < n_chunks; ++k) { const int i0 = (k * G + blockIdx.x) * FRAME_THREADS; if (i0 < N) total += (unsigned int)(min(FRAME_THREADS, N - i0) * 4) * 6u; }
            mbar_expect_tx(&s_mbar, total);
            for (int k = 0; k < n_chunks; ++k) {
                const int i0 = (k * G + blockIdx.x) * FRAME_THREADS;
                if (i0 >= N) continue;
                const unsigned int bytes = (unsigned int)(min(FRAME_THREADS, N - i0) * 4);
#pragma unroll
                for (int pl = 0; pl < 3; ++pl) {
                    tma_bulk_g2s(&s_stage[((pl) * K + k) * FRAME_THREADS], ia.vmap_curr + (size_t)pl * N + i0, bytes, &s_mbar);
                    tma_bulk_g2s(&s_stage[((3 + pl) * K + k) * FRAME_THREADS], ia.nmap_curr + (size_t)pl * N + i0, bytes, &s_mbar);
                }
            }
        }
        for (int k = 0; k < n_chunks; ++k) {
            const int idx = (k * G + blockIdx.x) * FRAME_THREADS + tid;
            const int o = k * FRAME_THREADS + tid;
            unsigned int meta = 0; float d1 = 0.f; short2 gr = make_short2(0, 0);
            if (idx < N) meta = rgb_precheck(a, idx, gr, d1);
            s_meta[o] = meta; s_d1[o] = d1; s_grad[o] = gr;
        }
        if (WITH_ICP) { mbar_wait(&s_mbar, stage_parity); stage_parity ^= 1u; }
        __syncthreads();

        for (int iter = 0; iter < p.iters[level]; ++iter, ++it) {
            // warp of this iteration from the running estimate (RGBDOdometry.cpp:209-231)
            if (tid == 0) build_warp(s_pose.Rt, a.Kfx, a.Kfy, a.Kcx, a.Kcy, s_w, s_w + 9);
            __syncthreads();
            const Mat33 krkinv = mat33_rows(s_w);
            const float3 kt = make_float3(s_w[9], s_w[10], s_w[11]);
            const Mat33 Rcurr = mat33_rows(s_pose.R);
            const float3 tcurr = make_float3(s_pose.t[0], s_pose.t[1], s_pose.t[2]);

            // ---------------- pass A ----------------
            float sum[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) sum[k] = 0.f;
            int cnt = 0, sig = 0;
            int cu0[RGBD_MAX_K], cv0[RGBD_MAX_K]; float cdiff[RGBD_MAX_K], cd0[RGBD_MAX_K]; bool cval[RGBD_MAX_K];
#pragma unroll
            for (int k = 0; k < RGBD_MAX_K; ++k) {
                cval[k] = false; cu0[k] = 0; cv0[k] = 0; cdiff[k] = 0.f; cd0[k] = 0.f;
                if (k < n_chunks) {
                    const int idx = (k * G + blockIdx.x) * FRAME_THREADS + tid;
                    const int o = k * FRAME_THREADS + tid;
                    if (idx < N) {
                        const unsigned int meta = s_meta[o];
                        if (meta & 1u) {
                            const int y = idx / cols, x = idx - y * cols;
                            int u0, v0; float d0, diff;
                            if (rgb_correspond(krkinv, kt, x, y, s_d1[o], (meta >> 8) & 0xffu, lastDepth, lastImage, cols, rows, maxDepthDelta, u0, v0, d0, diff)) {
                                cval[k] = true; cu0[k] = u0; cv0[k] = v0; cdiff[k] = diff; cd0[k] = d0;
                                cnt += 1; sig += (int)(diff * diff);
                            }
                        }
                        if (WITH_ICP) {
                            const IcpLevelArgs& ia = p.icp[level];
                            const int ps = K * FRAME_THREADS;
                            const float3 vc = make_float3(s_stage[o], s_stage[ps + o], s_stage[2 * ps + o]);
                            const float3 nc = make_float3(s_stage[3 * ps + o], s_stage[4 * ps + o], s_stage[5 * ps + o]);
                            icp_pixel(vc, nc, N, cols, rows, ia.vmap_g_prev, ia.nmap_g_prev, ia.k, Rcurr, tcurr, Rprev_inv, tprev, ia.dist_thres, ia.angle_thres, sum);
                        }
                    }
                }
            }
            // reduce pass A: ints (count, sigma) and, with ICP, the 29 float sums -> exchange 1 (lanes 0..28: ICP sums, 29 / 30: count / sigma)
            for (int o = 16; o > 0; o >>= 1) { cnt += __shfl_down_sync(0xffffffffu, cnt, o); sig += __shfl_down_sync(0xffffffffu, sig, o); }
            if (lane == 0) { s_cnt[wid][0] = cnt; s_cnt[wid][1] = sig; }
            if (WITH_ICP) { const float v = warp_transpose_sum(sum, lane); s_red[wid][lane] = v; }
            __syncthreads();
            if (wid == 0) {
                long long q = 0;
                if (WITH_ICP && lane < NSUM) {
                    float v = 0.f;
#pragma unroll
                    for (int w = 0; w < FRAME_THREADS / 32; ++w) v += s_red[w][lane];
                    q = to_fixed32(v);
                } else if (lane == 29 || lane == 30) {
                    int c = 0;
                    for (int w = 0; w < FRAME_THREADS / 32; ++w) c += s_cnt[w][lane - 29];
                    q = (long long)c << 8;
                }
                const bool active = (WITH_ICP && lane < NSUM) || lane == 29 || lane == 30;
                const long long tot = grid_sum_fixed(p.xwords, ex, lane, active, q, gs, (unsigned int)G, p.timeout);
                if (WITH_ICP && lane < NSUM) icp_total = from_fixed32(tot);
                if (lane == 29 || lane == 30) s_tot[lane - 29] = (int)(tot >> 8);
            }
            ++ex;
            __syncthreads();
            // Q3: sigmaVal = sqrt((float)sigma / rgbSize == 0 ? 1 : rgbSize)   (RGBDOdometry.cpp:253)
            const int rgb_count = s_tot[0], rgb_sigma = s_tot[1];
            const float sigma = (float)sqrt((double)(((float)rgb_sigma / rgb_count == 0) ? 1 : rgb_count));

            // ---------------- pass B ----------------
#pragma unroll
            for (int k = 0; k < 32; ++k) sum[k] = 0.f;
#pragma unroll
            for (int k = 0; k < RGBD_MAX_K; ++k) {
                if (k < n_chunks && cval[k]) {
                    const float z = cd0[k];
                    const float3 cloudPoint = make_float3((float)((cu0[k] - dcx) * z * invFx), (float)((cv0[k] - dcy) * z * invFy), z);
                    const short2 gr = s_grad[k * FRAME_THREADS + tid];
                    rgb_pixel_row(sigma, cdiff[k], gr.x, gr.y, cloudPoint, sobelScale, fx, fy, sum);
                }
            }
            { const float v = warp_transpose_sum(sum, lane); s_red[wid][lane] = v; }
            __syncthreads();
            if (wid == 0) {
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < FRAME_THREADS / 32; ++w) v += s_red[w][lane];
                // exchange 2: the photometric sums, two words per component (their range is not bounded by geometry, kt_frame.cuh)
                const double total = grid_sum_words_wide(p.xwords, ex, lane, v, gs, gs_lo, (unsigned int)G, p.timeout);
                // A = A_rgb + 100 A_icp, b = b_rgb + 10 b_icp in double (RGBDOdometry.cpp:316-321); the b sums are components
                // 6, 12, 17, 21, 24, 26 of the 27 (internal.h:101-106 order)
                double m = total;
                if (WITH_ICP) {
                    const bool is_b = (lane == 6) || (lane == 12) || (lane == 17) || (lane == 21) || (lane == 24) || (lane == 26);
                    m = fma(is_b ? 10.0 : 100.0, icp_total, m);
                }
                s_sumd[lane] = m;
                __syncwarp();
                if (lane == 0) {
                    double dA[36], db[6];
                    unpack_normal_equations(s_sumd, dA, db);
                    gauss_newton_update_fast(dA, db, s_pose.Rt, s_pose.Rp, s_pose.tp, s_pose.R, s_pose.t);
                }
                if (p.trace && blockIdx.x == 0 && it < 64) {            // the photometric part alone, like the reference's A_rgb / b_rgb
                    float* t = p.trace + (size_t)it * TRACE_STRIDE;
                    const float value = (float)total;              // component -> slot worked out once per launch (trace_a / trace_b): CTA 0 is on every exchange's critical path
                    if (trace_a >= 0) t[trace_a] = value;
                    if (trace_b >= 0) t[trace_b] = value;
                    if (lane == 0) { t[42] = (float)rgb_sigma; t[43] = (float)rgb_count; }
                }
            }
            ++ex;
            __syncthreads();
        }
    }
    frame_end(s_pose, it, p.st, p.host_pose, p.host_seq, p.timeout);
}

} // namespace

#define KT_GRID2D(cols, rows) dim3 block(32, 8), grid(div_up(cols, 32), div_up(rows, 8))

int short_depth_to_metres(const uint16_t* src, float* dst, int rows, int cols, int cut_off, cudaStream_t s)
{ KT_GRID2D(cols, rows); PreParams p = {src, dst, 0, rows, cols, rows, cols, cut_off}; preprocess_kernel<PRE_METRES><<<grid, block, 0, s>>>(p); KT_LAUNCH_CHECK(); return 0; }

int bgr_to_intensity(const uint8_t* rgb, uint8_t* dst, int rows, int cols, cudaStream_t s)
{ KT_GRID2D(cols, rows); PreParams p = {rgb, dst, 0, rows, cols, rows, cols, 0}; preprocess_kernel<PRE_INTENSITY><<<grid, block, 0, s>>>(p); KT_LAUNCH_CHECK(); return 0; }

int pyrdown_gauss_f(const float* src, float* dst, int srows, int scols, cudaStream_t s)
{ int dr = srows / 2, dc = scols / 2; KT_GRID2D(dc, dr); PreParams p = {src, dst, 0, dr, dc, srows, scols, 0}; preprocess_kernel<PRE_DOWN_F><<<grid, block, 0, s>>>(p); KT_LAUNCH_CHECK(); return 0; }

int pyrdown_uchar_gauss(const uint8_t* src, uint8_t* dst, int srows, int scols, cudaStream_t s)
{ int dr = srows / 2, dc = scols / 2; KT_GRID2D(dc, dr); PreParams p = {src, dst, 0, dr, dc, srows, scols, 0}; preprocess_kernel<PRE_DOWN_U8><<<grid, block, 0, s>>>(p); KT_LAUNCH_CHECK(); return 0; }

int derivative_images(const uint8_t* src, int16_t* dx, int16_t* dy, int rows, int cols, cudaStream_t s)
{ KT_GRID2D(cols, rows); PreParams p = {src, dx, dy, rows, cols, rows, cols, 0}; preprocess_kernel<PRE_GRADIENT><<<grid, block, 0, s>>>(p); KT_LAUNCH_CHECK(); return 0; }

int project_to_point_cloud(const float* depth, float* cloud, int rows, int cols, double fx, double fy, double cx, double cy, cudaStream_t s)
{
    KT_GRID2D(cols, rows);
    // projectToPointCloud passes 1.0f / fx with fx double (maps.cu:342): a double division
    project_points_kernel<<<grid, block, 0, s>>>(depth, (float3*)cloud, rows, cols, 1.0f / fx, 1.0f / fy, cx, cy);
    KT_LAUNCH_CHECK();
    return 0;
}

int rgb_residual(const RgbLevelArgs& a, OdomState* state, int* partials, int use_state_warp, cudaStream_t s)
{
    ResidualParams p; p.a = a; p.st = state; p.partials = partials;
    int grid = reduce_grid_for(a.rows * a.cols);
    residual_kernel<<<grid, RED_THREADS, 0, s>>>(p, use_state_warp);
    KT_LAUNCH_CHECK();
    return 0;
}

int rgb_iteration(const RgbLevelArgs& a, OdomState* state, float* partials, float* trace, int mode, float sigma_override, cudaStream_t s)
{
    RgbStepParams p; p.a = a; p.st = state; p.partials = partials; p.trace = trace; p.mode = mode; p.sigma_override = sigma_override;
    int grid = reduce_grid_for(a.rows * a.cols);
    rgb_step_kernel<<<grid, RED_THREADS, 0, s>>>(p);
    KT_LAUNCH_CHECK();
    return 0;
}


// Whole-frame RGB-D / ICP+RGB-D odometry.  Returns 1 (and launches nothing) when the image does not fit the shared-memory stage,
// in which case the caller falls back to the per-iteration kernels above.
int rgbd_frame(const IcpLevelArgs* icp_levels, const RgbLevelArgs* rgb_levels, const int* iters, int with_icp, const float* pose12_host, OdomState* state,
               unsigned long long* xwords_dev, float* trace, int* timeout_dev, float* host_pose, unsigned int host_seq, cudaStream_t s)
{
    RgbdFrameParams p;
    p.host_pose = host_pose; p.host_seq = host_seq;
    for (int l = 0; l < LEVELS; ++l) { p.icp[l] = icp_levels[l]; p.rgb[l] = rgb_levels[l]; p.iters[l] = iters[l]; }
    for (int k = 0; k < 12; ++k) p.pose12[k] = pose12_host[k];
    p.st = state; p.xwords = xwords_dev; p.trace = trace; p.timeout = timeout_dev; p.with_icp = with_icp;
    DeviceInfo& di = device_info();
    const int smem_optin = di.smem_optin;
    const int grid = frame_grid();
    int need_k = 0;
    for (int l = 0; l < LEVELS; ++l)
        if (iters[l] > 0) { int k = div_up(rgb_levels[l].rows * rgb_levels[l].cols, grid * FRAME_THREADS); if (k > need_k) need_k = k; }
    if (need_k > RGBD_MAX_K) return 1;
    const size_t bytes = (size_t)need_k * FRAME_THREADS * ((with_icp ? 6 * 4 : 0) + 12);
    if (smem_optin <= 0 || bytes > (size_t)(smem_optin - 8192)) return 1;
    if (!(di.configured & 2u)) {
        cudaFuncSetAttribute((const void*)rgbd_frame_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin - 8192);
        cudaFuncSetAttribute((const void*)rgbd_frame_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin - 8192);
        di.configured |= 2u;
    }
    p.stage_k = need_k;
    void* args[] = {&p};
    cudaError_t e = with_icp ? cudaLaunchCooperativeKernel((const void*)rgbd_frame_kernel<true>, dim3(grid), dim3(FRAME_THREADS), args, bytes, s)
                             : cudaLaunchCooperativeKernel((const void*)rgbd_frame_kernel<false>, dim3(grid), dim3(FRAME_THREADS), args, bytes, s);
    ++g_launches;
    if (e != cudaSuccess) return cuda_check(e, "cudaLaunchCooperativeKernel(rgbd_frame_kernel)", __FILE__, __LINE__);
    return 0;
}

} // namespace kt
