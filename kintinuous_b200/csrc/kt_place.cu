// kintinuous_b200 -- place-recognition kernels behind kt_detect_loops (kt_tracker.cu) and the kt_op_* entry points.
//
// Stands in for (reference, src/backend/): DLoopDetector's retrieval with the DBoW2 vocabulary (PlaceRecognition.cpp:51-98) -- here an
// EXACT exhaustive ratio test against every stored keyframe, no vocabulary --, Surf3DTools::surfMatch3D's FLANN 2-NN (Surf3DTools.h:105-274,
// here exact), Surf3DTools::calculate3dPointsSURF's depth lookup and PNPSolver::getRelativePose (PNPSolver.cpp, cv::solvePnPRansac), and
// DepthCamera::convertToXYZPointCloud for the fitness check (the voxel grid and nearest-neighbour search are kt_slice.cu's).
//   match_ratio   one thread per database row (one OLD feature, the reference's direction) holds its descriptor in registers and streams
//                 the query (NEW keyframe) descriptors through shared memory: d = sum_k (a_k - b_k)^2 in ascending k with FMA, so a row's
//                 result does not depend on the tiling; the two smallest (ties: lower index) and the test d1 < ratio * d2.  Pass counts per
//                 keyframe are integer sums, deterministic in any order.  FP32 FFMA, no tensor cores (exactness first).
//   pnp_ransac    ONE launch: a CTA per hypothesis -- 3 matches drawn by a counter-based hash of (seed, hypothesis, draw), the pose from
//                 their 3-D <-> 3-D correspondence (Horn's quaternion form of Kabsch, FP64; both keypoints have depth, so no P3P), inliers =
//                 reprojection into the old image <= threshold px --, then the last CTA to finish picks the most inliers (ties: lower
//                 hypothesis), refines that pose by FP64 Gauss-Newton on the reprojection error of its inliers (kt_solve.cuh's 6 x 6 LDL^T)
//                 and recomputes the inliers.  Every sum has a fixed order: bitwise reproducible.
#include "kt_ops.h"
#include "kt_solve.cuh"
#include "kt_place.hpp"
#include "../../include/kintinuous_b200.h"

namespace kt {

namespace {

enum { MR_THREADS = 128, MR_TILE = 32, PNP_THREADS = 128 };

__global__ void keypoints_3d_kernel(const float* __restrict__ kp, const int* __restrict__ n_dev, int max_n, const uint16_t* __restrict__ depth,
                                    int rows, int cols, Intr k, float* __restrict__ xyz)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= max_n) return;
    float o[3] = {qnan(), qnan(), qnan()};
    if (i < *n_dev) {
        const float x = kp[(size_t)i * 6], y = kp[(size_t)i * 6 + 1];
        const int ui = (int)floorf(x + 0.5f), vi = (int)floorf(y + 0.5f);
        // kt_place.hpp place_lookup_3d: +-0.5 px strict, depth != 0, z < 10 m
        if (fabsf((float)ui - x) < 0.5f && fabsf((float)vi - y) < 0.5f && ui >= 0 && vi >= 0 && ui < cols && vi < rows) {
            const uint16_t d = depth[(size_t)vi * cols + ui];
            const float z = __fdiv_rn((float)d, 1000.f);
            if (d != 0 && z < 10.f) {
                o[0] = __fdiv_rn(__fmul_rn(z, __fsub_rn((float)ui, k.cx)), k.fx);
                o[1] = __fdiv_rn(__fmul_rn(z, __fsub_rn((float)vi, k.cy)), k.fy);
                o[2] = z;
            }
        }
    }
    xyz[(size_t)i * 3] = o[0]; xyz[(size_t)i * 3 + 1] = o[1]; xyz[(size_t)i * 3 + 2] = o[2];
}

__global__ void __launch_bounds__(MR_THREADS) match_ratio_kernel(const float* __restrict__ db, int n_rows, int stride, const int* __restrict__ seg_count,
                                                                 const float* __restrict__ q, const int* __restrict__ n_query_dev, int q_cap, float ratio,
                                                                 int* __restrict__ best, float* __restrict__ d1o, float* __restrict__ d2o,
                                                                 unsigned char* __restrict__ pass)
{
    __shared__ float4 s_q[MR_TILE][16];
    const int row = blockIdx.x * MR_THREADS + threadIdx.x;
    const int nq = min(*n_query_dev, q_cap);
    const bool valid = row < n_rows && (row % stride) < seg_count[row / stride];
    float a[64];
    if (valid) {
        const float4* src = reinterpret_cast<const float4*>(db + (size_t)row * 64);
#pragma unroll
        for (int k = 0; k < 16; ++k) { const float4 v = __ldg(src + k); a[4 * k] = v.x; a[4 * k + 1] = v.y; a[4 * k + 2] = v.z; a[4 * k + 3] = v.w; }
    } else {
#pragma unroll
        for (int k = 0; k < 64; ++k) a[k] = 0.f;
    }
    float d1 = 3.0e38f, d2 = 3.0e38f; int j1 = -1;
    for (int base = 0; base < nq; base += MR_TILE) {
        __syncthreads();
        for (int t = threadIdx.x; t < MR_TILE * 16; t += MR_THREADS) {
            const int j = base + t / 16;
            s_q[t / 16][t % 16] = j < nq ? __ldg(reinterpret_cast<const float4*>(q + (size_t)j * 64) + (t % 16)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncthreads();
        const int nt = min(MR_TILE, nq - base);
        for (int jj = 0; jj < nt; ++jj) {
            float d = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const float4 b = s_q[jj][k];
                float e;
                e = a[4 * k] - b.x; d = __fmaf_rn(e, e, d);
                e = a[4 * k + 1] - b.y; d = __fmaf_rn(e, e, d);
                e = a[4 * k + 2] - b.z; d = __fmaf_rn(e, e, d);
                e = a[4 * k + 3] - b.w; d = __fmaf_rn(e, e, d);
            }
            if (d < d1) { d2 = d1; d1 = d; j1 = base + jj; }
            else if (d < d2) d2 = d;
        }
    }
    if (row < n_rows) {
        const bool ok = valid && nq >= 2 && d1 < __fmul_rn(ratio, d2);
        best[row] = valid ? j1 : -1; d1o[row] = d1; d2o[row] = d2; pass[row] = ok ? 1 : 0;
    }
}

__global__ void seg_passes_kernel(const unsigned char* __restrict__ pass, int stride, int* __restrict__ out)
{
    __shared__ int s[256];
    const unsigned char* p = pass + (size_t)blockIdx.x * stride;
    int c = 0;
    for (int i = threadIdx.x; i < stride; i += blockDim.x) c += p[i];
    s[threadIdx.x] = c;
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) { if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) out[blockIdx.x] = s[0];
}

// ---- PnP RANSAC ----
__device__ __forceinline__ unsigned int hash3(unsigned long long seed, unsigned int h, unsigned int k)      // splitmix64 of the counter
{
    unsigned long long z = seed + 0x9e3779b97f4a7c15ull * ((((unsigned long long)h) << 20) + k + 1);
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return (unsigned int)((z ^ (z >> 31)) >> 32);
}

// largest eigenpair of a symmetric 4 x 4 matrix by cyclic Jacobi (FP64)
__device__ void jacobi4_max(double A[4][4], double* v)
{
    double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0;
        for (int p = 0; p < 4; ++p) for (int q = p + 1; q < 4; ++q) off += A[p][q] * A[p][q];
        if (off < 1e-30) break;
        for (int p = 0; p < 4; ++p)
            for (int q = p + 1; q < 4; ++q) {
                if (fabs(A[p][q]) < 1e-300) continue;
                const double th = 0.5 * (A[q][q] - A[p][p]) / A[p][q];
                const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 4; ++k) { const double akp = A[k][p], akq = A[k][q]; A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq; }
                for (int k = 0; k < 4; ++k) { const double apk = A[p][k], aqk = A[q][k]; A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk; }
                for (int k = 0; k < 4; ++k) { const double vkp = V[k][p], vkq = V[k][q]; V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq; }
            }
    }
    int b = 0;
    for (int k = 1; k < 4; ++k) if (A[k][k] > A[b][b]) b = k;
    for (int k = 0; k < 4; ++k) v[k] = V[k][b];
}

// R (row-major), t with R a + t ~ b for the three pairs (a = new, b = old); false for a degenerate sample
__device__ bool kabsch3(const float* __restrict__ pa, const float* __restrict__ pb, const int* id, double* R, double* t)
{
    double ca[3] = {0, 0, 0}, cb[3] = {0, 0, 0};
    for (int m = 0; m < 3; ++m) for (int e = 0; e < 3; ++e) { ca[e] += pa[id[m] * 3 + e] / 3.0; cb[e] += pb[id[m] * 3 + e] / 3.0; }
    double S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int m = 0; m < 3; ++m)
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) S[i][j] += (pa[id[m] * 3 + i] - ca[i]) * (pb[id[m] * 3 + j] - cb[j]);
    // the sample's triangle must not be degenerate (area^2 > 1e-8 m^4)
    double u[3], w[3];
    for (int e = 0; e < 3; ++e) { u[e] = pa[id[1] * 3 + e] - pa[id[0] * 3 + e]; w[e] = pa[id[2] * 3 + e] - pa[id[0] * 3 + e]; }
    const double cx = u[1] * w[2] - u[2] * w[1], cy = u[2] * w[0] - u[0] * w[2], cz = u[0] * w[1] - u[1] * w[0];
    if (cx * cx + cy * cy + cz * cz < 4e-8) return false;
    double N[4][4] = {
        {S[0][0] + S[1][1] + S[2][2], S[1][2] - S[2][1], S[2][0] - S[0][2], S[0][1] - S[1][0]},
        {S[1][2] - S[2][1], S[0][0] - S[1][1] - S[2][2], S[0][1] + S[1][0], S[2][0] + S[0][2]},
        {S[2][0] - S[0][2], S[0][1] + S[1][0], -S[0][0] + S[1][1] - S[2][2], S[1][2] + S[2][1]},
        {S[0][1] - S[1][0], S[2][0] + S[0][2], S[1][2] + S[2][1], -S[0][0] - S[1][1] + S[2][2]}};
    double q[4];
    jacobi4_max(N, q);
    const double qw = q[0], qx = q[1], qy = q[2], qz = q[3];
    R[0] = qw * qw + qx * qx - qy * qy - qz * qz; R[1] = 2 * (qx * qy - qw * qz); R[2] = 2 * (qx * qz + qw * qy);
    R[3] = 2 * (qx * qy + qw * qz); R[4] = qw * qw - qx * qx + qy * qy - qz * qz; R[5] = 2 * (qy * qz - qw * qx);
    R[6] = 2 * (qx * qz - qw * qy); R[7] = 2 * (qy * qz + qw * qx); R[8] = qw * qw - qx * qx - qy * qy + qz * qz;
    for (int e = 0; e < 3; ++e) t[e] = cb[e] - (R[3 * e] * ca[0] + R[3 * e + 1] * ca[1] + R[3 * e + 2] * ca[2]);
    return true;
}

// reprojection of new point i into the old image; false behind the camera
__device__ __forceinline__ bool reproject(const double* R, const double* t, const float* __restrict__ pa, int i, const Intr& k, double* X, double* uv)
{
    const double a0 = pa[i * 3], a1 = pa[i * 3 + 1], a2 = pa[i * 3 + 2];
    for (int e = 0; e < 3; ++e) X[e] = R[3 * e] * a0 + R[3 * e + 1] * a1 + R[3 * e + 2] * a2 + t[e];
    if (!(X[2] > 0)) return false;
    uv[0] = (double)k.fx * X[0] / X[2] + (double)k.cx; uv[1] = (double)k.fy * X[1] / X[2] + (double)k.cy;
    return true;
}
__device__ __forceinline__ bool is_inlier(const double* R, const double* t, const float* __restrict__ pa, const float* __restrict__ uv_old, int i, const Intr& k, double thr2)
{
    double X[3], uv[2];
    if (!reproject(R, t, pa, i, k, X, uv)) return false;
    const double du = uv[0] - uv_old[2 * i], dv = uv[1] - uv_old[2 * i + 1];
    return du * du + dv * dv <= thr2;
}

// fixed-order block sum of n doubles per thread into s (n x PNP_THREADS), result in s[k * PNP_THREADS]
__device__ void block_sum(double* s, int n)
{
    for (int o = PNP_THREADS / 2; o > 0; o >>= 1) {
        __syncthreads();
        if ((int)threadIdx.x < o) for (int k = 0; k < n; ++k) s[k * PNP_THREADS + threadIdx.x] += s[k * PNP_THREADS + threadIdx.x + o];
    }
    __syncthreads();
}

__global__ void __launch_bounds__(PNP_THREADS) pnp_ransac_kernel(const PnpArgs a, int* __restrict__ counts, double* __restrict__ hyps,
                                                                  unsigned int* __restrict__ counter, double* __restrict__ pose12,
                                                                  unsigned char* __restrict__ inliers, int* __restrict__ n_inliers)
{
    __shared__ double s_pose[12];
    __shared__ int s_ok;
    __shared__ int s_cnt[PNP_THREADS];
    __shared__ bool s_last;
    extern __shared__ double s_red[];                         // 27 x PNP_THREADS
    const int h = blockIdx.x, n = a.n;
    const double thr2 = (double)a.threshold_px * a.threshold_px;
    if (threadIdx.x == 0) {
        int id[3] = {0, 0, 0};
        s_ok = 0;
        for (int attempt = 0; attempt < 64 && !s_ok; ++attempt) {
            for (int m = 0; m < 3; ++m) id[m] = (int)(hash3(a.seed, (unsigned int)h, (unsigned int)(attempt * 3 + m)) % (unsigned int)n);
            if (id[0] == id[1] || id[0] == id[2] || id[1] == id[2]) continue;
            if (kabsch3(a.p_new, a.p_old, id, s_pose, s_pose + 9)) s_ok = 1;
        }
    }
    __syncthreads();
    int c = 0;
    if (s_ok) for (int i = threadIdx.x; i < n; i += PNP_THREADS) c += is_inlier(s_pose, s_pose + 9, a.p_new, a.uv_old, i, a.k, thr2) ? 1 : 0;
    s_cnt[threadIdx.x] = c;
    __syncthreads();
    for (int o = PNP_THREADS / 2; o > 0; o >>= 1) { if ((int)threadIdx.x < o) s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) {
        counts[h] = s_ok ? s_cnt[0] : -1;
        for (int e = 0; e < 12; ++e) hyps[(size_t)h * 12 + e] = s_pose[e];
        __threadfence();
        s_last = atomicAdd(counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // the last CTA: best hypothesis (most inliers, ties to the lower index), refinement, final inliers
    if (threadIdx.x == 0) {
        int b = 0;
        for (int k = 1; k < (int)gridDim.x; ++k) if (((volatile int*)counts)[k] > ((volatile int*)counts)[b]) b = k;
        s_ok = ((volatile int*)counts)[b];
        for (int e = 0; e < 12; ++e) s_pose[e] = ((volatile double*)hyps)[(size_t)b * 12 + e];
        *counter = 0;
    }
    __syncthreads();
    if (s_ok < 0) {
        for (int i = threadIdx.x; i < n; i += PNP_THREADS) inliers[i] = 0;
        if (threadIdx.x == 0) { *n_inliers = 0; for (int e = 0; e < 12; ++e) pose12[e] = (e % 4 == 0 && e < 9) ? 1.0 : 0.0; }
        return;
    }
    // inliers of the best hypothesis: the fixed set of the Gauss-Newton refinement
    for (int i = threadIdx.x; i < n; i += PNP_THREADS) inliers[i] = is_inlier(s_pose, s_pose + 9, a.p_new, a.uv_old, i, a.k, thr2) ? 1 : 0;
    __syncthreads();
    if (s_ok >= 6) {
        for (int it = 0; it < 10; ++it) {
            double acc[27];
            for (int k = 0; k < 27; ++k) acc[k] = 0;
            for (int i = threadIdx.x; i < n; i += PNP_THREADS) {
                if (!inliers[i]) continue;
                double X[3], uv[2];
                if (!reproject(s_pose, s_pose + 9, a.p_new, i, a.k, X, uv)) continue;
                const double iz = 1.0 / X[2], fx = a.k.fx, fy = a.k.fy;
                const double r0 = uv[0] - a.uv_old[2 * i], r1 = uv[1] - a.uv_old[2 * i + 1];
                // d(uv)/dX, X' = X + w x X + v: dX/dv = I, dX/dw = -[X]x
                const double P0[3] = {fx * iz, 0.0, -fx * X[0] * iz * iz}, P1[3] = {0.0, fy * iz, -fy * X[1] * iz * iz};
                double J0[6], J1[6];
                for (int e = 0; e < 3; ++e) { J0[e] = P0[e]; J1[e] = P1[e]; }
                // dX/dw = -[X]x, whose columns are (0, -X2, X1), (X2, 0, -X0), (-X1, X0, 0): the rotation block is X x P
                J0[3] = X[1] * P0[2] - X[2] * P0[1]; J0[4] = X[2] * P0[0] - X[0] * P0[2]; J0[5] = X[0] * P0[1] - X[1] * P0[0];
                J1[3] = X[1] * P1[2] - X[2] * P1[1]; J1[4] = X[2] * P1[0] - X[0] * P1[2]; J1[5] = X[0] * P1[1] - X[1] * P1[0];
                int q = 0;
                for (int r = 0; r < 6; ++r) for (int cc = r; cc < 6; ++cc) acc[q++] += J0[r] * J0[cc] + J1[r] * J1[cc];
                for (int r = 0; r < 6; ++r) acc[21 + r] += J0[r] * r0 + J1[r] * r1;
            }
            for (int k = 0; k < 27; ++k) s_red[k * PNP_THREADS + threadIdx.x] = acc[k];
            block_sum(s_red, 27);
            if (threadIdx.x == 0) {
                double A[36], b[6], x[6];
                int q = 0;
                for (int r = 0; r < 6; ++r) for (int cc = r; cc < 6; ++cc) { A[r * 6 + cc] = A[cc * 6 + r] = s_red[(q++) * PNP_THREADS]; }
                for (int r = 0; r < 6; ++r) b[r] = -s_red[(21 + r) * PNP_THREADS];
                ldlt6_solve(A, b, x);
                double dR[9];
                rodrigues(x + 3, dR);
                double Rn[9], tn[3];
                for (int i = 0; i < 3; ++i) {
                    for (int j = 0; j < 3; ++j) Rn[i * 3 + j] = dR[i * 3] * s_pose[j] + dR[i * 3 + 1] * s_pose[3 + j] + dR[i * 3 + 2] * s_pose[6 + j];
                    tn[i] = dR[i * 3] * s_pose[9] + dR[i * 3 + 1] * s_pose[10] + dR[i * 3 + 2] * s_pose[11] + x[i];
                }
                for (int e = 0; e < 9; ++e) s_pose[e] = Rn[e];
                for (int e = 0; e < 3; ++e) s_pose[9 + e] = tn[e];
            }
            __syncthreads();
        }
    }
    c = 0;
    for (int i = threadIdx.x; i < n; i += PNP_THREADS) { const bool in = is_inlier(s_pose, s_pose + 9, a.p_new, a.uv_old, i, a.k, thr2); inliers[i] = in ? 1 : 0; c += in ? 1 : 0; }
    s_cnt[threadIdx.x] = c;
    __syncthreads();
    for (int o = PNP_THREADS / 2; o > 0; o >>= 1) { if ((int)threadIdx.x < o) s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) { *n_inliers = s_cnt[0]; for (int e = 0; e < 12; ++e) pose12[e] = s_pose[e]; }
}

__global__ void depth_to_cloud_kernel(const uint16_t* __restrict__ depth, int rows, int cols, Intr k, kt_point_xyzrgb* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * cols) return;
    const int u = i % cols, v = i / cols;
    const uint16_t d = depth[i];
    kt_point_xyzrgb p;
    const float z = __fdiv_rn((float)d, 1000.f);
    p.x = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, k.cx), z), k.fx); p.y = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, k.cy), z), k.fy); p.z = z; p._pad0 = 1.f;
    p.b = p.g = p.r = 0; p.a = d != 0 ? 1 : 0;             // alpha = validity: the voxel grid's weight cull (1) drops the holes
    for (int e = 0; e < 12; ++e) p._pad1[e] = 0;
    out[i] = p;
}

} // namespace

int keypoints_3d(const float* kp, const int* n_dev, int max_n, const uint16_t* depth, int rows, int cols, const Intr& k, float* xyz, cudaStream_t s)
{
    if (max_n <= 0) return 0;
    keypoints_3d_kernel<<<div_up(max_n, 128), 128, 0, s>>>(kp, n_dev, max_n, depth, rows, cols, k, xyz);
    KT_LAUNCH_CHECK();
    return 0;
}

int match_ratio(const float* db, int n_seg, int stride, const int* seg_count_dev, const float* q, const int* n_query_dev, int q_cap, float ratio,
                int* best, float* d1, float* d2, unsigned char* pass, int* seg_passes, cudaStream_t s)
{
    if (n_seg <= 0 || stride <= 0) return 0;
    const long long rows = (long long)n_seg * stride;
    if (rows > (1ll << 31) - MR_THREADS) { set_error("match_ratio: %lld database rows", rows); return KT_ERR_INVALID; }
    match_ratio_kernel<<<div_up((int)rows, MR_THREADS), MR_THREADS, 0, s>>>(db, (int)rows, stride, seg_count_dev, q, n_query_dev, q_cap, ratio, best, d1, d2, pass);
    KT_LAUNCH_CHECK();
    if (seg_passes) {
        seg_passes_kernel<<<n_seg, 256, 0, s>>>(pass, stride, seg_passes);
        KT_LAUNCH_CHECK();
    }
    return 0;
}

int pnp_ransac(const PnpArgs& a, PnpWorkspace* ws, double* pose12, unsigned char* inliers, int* n_inliers, cudaStream_t s)
{
    if (a.n < 3 || a.iterations < 1) { set_error("pnp_ransac: need at least 3 matches and 1 iteration"); return KT_ERR_INVALID; }
    const size_t it = (size_t)a.iterations;
    int r;
    if ((r = ws->counts.grow(it, it, "pnp inlier counts")) || (r = ws->hyps.grow(12 * it, 12 * it, "pnp hypotheses"))) return r;
    if (!ws->counter.get()) {
        if ((r = ws->counter.grow(1, 1, "pnp counter"))) return r;
        KT_CUDA(cudaMemset(ws->counter.get(), 0, sizeof(unsigned int)));
    }
    pnp_ransac_kernel<<<a.iterations, PNP_THREADS, 27 * PNP_THREADS * sizeof(double), s>>>(a, ws->counts.get(), ws->hyps.get(), ws->counter.get(), pose12, inliers, n_inliers);
    KT_LAUNCH_CHECK();
    return 0;
}

int depth_to_cloud(const uint16_t* depth, int rows, int cols, const Intr& k, void* cloud, cudaStream_t s)
{
    depth_to_cloud_kernel<<<div_up(rows * cols, 256), 256, 0, s>>>(depth, rows, cols, k, (kt_point_xyzrgb*)cloud);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
