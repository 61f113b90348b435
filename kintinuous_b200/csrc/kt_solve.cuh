// kintinuous_b200 -- on-device Gauss-Newton step: 6x6 solve, se(3) exponential and pose update.
//
// Replaces the HOST side of every odometry iteration in the reference, so that the coarse-to-fine
// loop runs without a device->host round trip (the reference does sync + 116-byte D2H + host LDLT
// 19 times per frame, SURVEY.md section 3.2):
//   unpack 27 sums -> A (6x6, symmetric), b (6)          cuda/reduce.cu:404-415
//   x = A.ldlt().solve(b) in double                       ICPOdometry.cpp:127-131, RGBDOdometry.cpp:316-326
//   currRt = [Rodrigues(x[3..5]) | x[0..2]]               OdometryProvider.h:54-68 (cv::Rodrigues, 64F)
//   resultRt = currRt * resultRt                          ICPOdometry.cpp:144
//   [Rcurr|tcurr] = [Rprev|tprev] * inverse([rot|trans])  ICPOdometry.cpp:146-178 (Eigen::Isometry3f, float)
// One thread executes this (a few hundred dependent FP64 ops, ~1-2 us); it is called by the last
// CTA of the reduction kernel.
#pragma once
#include "kt_ops.h"
#include <float.h>

// The functions of this header also compile for the HOST (tests/cpp/solve_host.cu, run by `pytest -m "not gpu"` against numpy / cv2 / the
// oracle): KT_HD = __host__ __device__, and the IEEE round-to-nearest intrinsics fall back to plain operators there (x86-64 SSE
// arithmetic is IEEE and gcc does not contract without an FMA target).  Device code generation is unchanged by this.
#define KT_HD __host__ __device__
#ifdef __CUDA_ARCH__
#define KT_FMUL(a, b) __fmul_rn((a), (b))
#define KT_FADD(a, b) __fadd_rn((a), (b))
#define KT_FSUB(a, b) __fsub_rn((a), (b))
#define KT_FDIV(a, b) __fdiv_rn((a), (b))
#else
#define KT_FMUL(a, b) ((a) * (b))
#define KT_FADD(a, b) ((a) + (b))
#define KT_FSUB(a, b) ((a) - (b))
#define KT_FDIV(a, b) ((a) / (b))
#endif

namespace kt {

// sums: 27 upper-triangular products in the order aa ab ac ad ae af ag bb ... fg (cuda/internal.h:101-106), unpacked like
// cuda/reduce.cu:404-415.  T = float (the reference's host copy) or double (the whole-frame kernels' exact totals); fully unrolled, so
// that the indices are constants and A, b stay in registers.
template <typename T>
KT_HD __forceinline__ void unpack_normal_equations(const T* sums, T* A, T* b)
{
    int shift = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = i; j < 7; ++j) {
            const T value = sums[shift++];
            if (j == 6) b[i] = value;
            else A[j * 6 + i] = A[i * 6 + j] = value;
        }
}

// x = A^-1 b for the symmetric positive (semi-)definite 6x6 normal matrix, LDL^T in FP64, fully unrolled so that the
// whole factorisation lives in registers (a local-memory version with pivot swaps costs ~18 us of dependent latency on one
// thread; this one ~1 us).  Eigen::LDLT pivots on the largest diagonal entry; for an SPD matrix both orders are backward
// stable and the solutions agree to ~cond(A) * 1e-16, far below the float pose they are rounded to.  A vanishing pivot
// (degenerate geometry, e.g. no inliers) contributes 0 to the solution, which is what Eigen's solve does with its tolerance.
KT_HD __forceinline__ void ldlt6_solve(const double* Ain, const double* bin, double* x)
{
    double a[6][6];
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) a[i][j] = Ain[i * 6 + j];
    double dinv[6];
    double scale = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) scale = fmax(scale, fabs(a[i][i]));
    const double tiny = scale * 1e-30 + DBL_MIN;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double d = a[k][k];
        const double inv = (fabs(d) > tiny) ? 1.0 / d : 0.0;
        dinv[k] = inv;
        double col[6], l[6];
#pragma unroll
        for (int i = k + 1; i < 6; ++i) { col[i] = a[i][k]; l[i] = col[i] * inv; }      // L(i,k) = A(i,k) / d_k
#pragma unroll
        for (int i = k + 1; i < 6; ++i)
#pragma unroll
            for (int j = k + 1; j <= i; ++j) a[i][j] -= l[i] * col[j];                    // A(i,j) -= L(i,k) d_k L(j,k)
#pragma unroll
        for (int i = k + 1; i < 6; ++i) a[i][k] = l[i];
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double v = bin[i];
#pragma unroll
        for (int j = 0; j < i; ++j) v -= a[i][j] * y[j];
        y[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] *= dinv[i];
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        double v = y[i];
#pragma unroll
        for (int j = i + 1; j < 6; ++j) v -= a[j][i] * y[j];
        y[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) x[i] = y[i];
}

// cv::Rodrigues, rotation vector -> matrix, double (OpenCV 2.4.9 semantics)
KT_HD inline void rodrigues(const double* r, double* R)
{
    double rx = r[0], ry = r[1], rz = r[2];
    double theta = sqrt(rx * rx + ry * ry + rz * rz);
    if (theta < DBL_EPSILON) {
        for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
        return;
    }
    double s, c;
    sincos(theta, &s, &c);
    const double c1 = 1.0 - c;
    double itheta = 1.0 / theta;
    rx *= itheta; ry *= itheta; rz *= itheta;
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    double rx_[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    for (int k = 0; k < 9; ++k) R[k] = c * I[k] + c1 * rrt[k] + s * rx_[k];
}

KT_HD __forceinline__ void mat3f_inverse(const float* m, float* r)   // Eigen 3x3 inverse (cofactors / det)
{
#define KT_M(i, j) m[(i) * 3 + (j)]
#define KT_COF(i, j) (KT_M(((i) + 1) % 3, ((j) + 1) % 3) * KT_M(((i) + 2) % 3, ((j) + 2) % 3) - KT_M(((i) + 1) % 3, ((j) + 2) % 3) * KT_M(((i) + 2) % 3, ((j) + 1) % 3))
    float c00 = KT_FSUB(KT_FMUL(KT_M(1, 1), KT_M(2, 2)), KT_FMUL(KT_M(1, 2), KT_M(2, 1)));
    float c10 = KT_FSUB(KT_FMUL(KT_M(2, 1), KT_M(0, 2)), KT_FMUL(KT_M(2, 2), KT_M(0, 1)));
    float c20 = KT_FSUB(KT_FMUL(KT_M(0, 1), KT_M(1, 2)), KT_FMUL(KT_M(0, 2), KT_M(1, 1)));
    float det = KT_FADD(KT_FADD(KT_FMUL(c00, KT_M(0, 0)), KT_FMUL(c10, KT_M(1, 0))), KT_FMUL(c20, KT_M(2, 0)));
    float invdet = KT_FDIV(1.0f, det);
    float c01 = KT_FSUB(KT_FMUL(KT_M(1, 2), KT_M(2, 0)), KT_FMUL(KT_M(1, 0), KT_M(2, 2)));
    float c11 = KT_FSUB(KT_FMUL(KT_M(2, 2), KT_M(0, 0)), KT_FMUL(KT_M(2, 0), KT_M(0, 2)));
    float c21 = KT_FSUB(KT_FMUL(KT_M(0, 2), KT_M(1, 0)), KT_FMUL(KT_M(0, 0), KT_M(1, 2)));
    float c02 = KT_FSUB(KT_FMUL(KT_M(1, 0), KT_M(2, 1)), KT_FMUL(KT_M(1, 1), KT_M(2, 0)));
    float c12 = KT_FSUB(KT_FMUL(KT_M(2, 0), KT_M(0, 1)), KT_FMUL(KT_M(2, 1), KT_M(0, 0)));
    float c22 = KT_FSUB(KT_FMUL(KT_M(0, 0), KT_M(1, 1)), KT_FMUL(KT_M(0, 1), KT_M(1, 0)));
    r[0] = KT_FMUL(c00, invdet); r[1] = KT_FMUL(c10, invdet); r[2] = KT_FMUL(c20, invdet);
    r[3] = KT_FMUL(c01, invdet); r[4] = KT_FMUL(c11, invdet); r[5] = KT_FMUL(c21, invdet);
    r[6] = KT_FMUL(c02, invdet); r[7] = KT_FMUL(c12, invdet); r[8] = KT_FMUL(c22, invdet);
#undef KT_COF
#undef KT_M
}

// IEEE (non-contracted) float helpers: the reference does this part on the HOST CPU, without FMA.
KT_HD __forceinline__ float dot3_rn(float a0, float a1, float a2, float b0, float b1, float b2)
{
    return KT_FADD(KT_FADD(KT_FMUL(a0, b0), KT_FMUL(a1, b1)), KT_FMUL(a2, b2));
}

// Solve for the increment and update resultRt (4x4 double) and the float pose (Rcurr, tcurr) given (Rprev, tprev).
KT_HD __forceinline__ void gauss_newton_update_p(const double* dA, const double* db, double* resultRt,
                                                      const float* Rp, const float* tprev, float* Rcurr, float* tcurr, long long* stamps = 0)
{
    double x[6];
    ldlt6_solve(dA, db, x);
#ifdef __CUDA_ARCH__
    if (stamps) stamps[0] = clock64();            // debug (tools/icp_prof.py)
#endif
    double R[9];
    rodrigues(x + 3, R);
#ifdef __CUDA_ARCH__
    if (stamps) stamps[1] = clock64();
#endif
    const double cur[16] = {R[0], R[1], R[2], x[0], R[3], R[4], R[5], x[1], R[6], R[7], R[8], x[2], 0, 0, 0, 1};
    double res[16];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double s = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) s += cur[i * 4 + k] * resultRt[k * 4 + j];
            res[i * 4 + j] = s;
        }
#pragma unroll
    for (int k = 0; k < 16; ++k) resultRt[k] = res[k];
    // float part (Eigen::Isometry3f): inverse of [rot|tr] is [rot^T | -rot^T tr]; then Rprev * that.
    float rot[9], tr[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) rot[i * 3 + j] = (float)res[i * 4 + j];
        tr[i] = (float)res[i * 4 + 3];
    }
    float tinv[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) tinv[i] = -dot3_rn(rot[0 * 3 + i], rot[1 * 3 + i], rot[2 * 3 + i], tr[0], tr[1], tr[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j)   // (Rprev * rot^T)(i,j) = sum_k Rprev(i,k) * rot(j,k)
            Rcurr[i * 3 + j] = dot3_rn(Rp[i * 3 + 0], Rp[i * 3 + 1], Rp[i * 3 + 2], rot[j * 3 + 0], rot[j * 3 + 1], rot[j * 3 + 2]);
        tcurr[i] = KT_FADD(dot3_rn(Rp[i * 3 + 0], Rp[i * 3 + 1], Rp[i * 3 + 2], tinv[0], tinv[1], tinv[2]), tprev[i]);
    }
}


// ------------------------------------------------------------------------------------------------------------------
// Latency-trimmed form of the same step, used inside the whole-frame kernels where ONE thread's dependent FP64 chain sits on the
// critical path of every Gauss-Newton iteration (19 per frame).  Same mathematics, same FP64 precision class:
//   * 1/d_k of the LDL^T pivots: hardware reciprocal seed (rcp.approx.ftz.f64, ~2^-20) + three Newton steps (error squares each
//     step: below 2^-53 after two; the third makes it robust) instead of the IEEE division subroutine -- on the device only; the
//     host build keeps the plain division;
//   * Rodrigues for |r|^2 <= 0.25 (|r| <= 0.5 rad = 28 degrees per ITERATION; tracking increments are < 0.05): the series of
//     sin(t)/t and (1 - cos t)/t^2 in t^2 (terms to t^18 / 19!, truncation < 1e-19) -- no sqrt, no division, no sincos; larger
//     rotations take the closed form above;
//   * the 4x4 product keeps only the three rows that are not (0 0 0 1).
// tests/test_device_solve_on_host.py runs both forms against numpy / cv2.Rodrigues.
KT_HD __forceinline__ double fast_rcp(double d)
{
#ifdef __CUDA_ARCH__
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
    r = fma(r, fma(-d, r, 1.0), r);
    r = fma(r, fma(-d, r, 1.0), r);
    r = fma(r, fma(-d, r, 1.0), r);
    return r;
#else
    return 1.0 / d;
#endif
}

KT_HD __forceinline__ void ldlt6_solve_fast(const double* Ain, const double* bin, double* x)
{
    double a[6][6];
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) a[i][j] = Ain[i * 6 + j];
    double dinv[6];
    double scale = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) scale = fmax(scale, fabs(a[i][i]));
    const double tiny = scale * 1e-30 + DBL_MIN;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double d = a[k][k];
        const double inv = (fabs(d) > tiny) ? fast_rcp(d) : 0.0;
        dinv[k] = inv;
        double col[6], l[6];
#pragma unroll
        for (int i = k + 1; i < 6; ++i) { col[i] = a[i][k]; l[i] = col[i] * inv; }
#pragma unroll
        for (int i = k + 1; i < 6; ++i)
#pragma unroll
            for (int j = k + 1; j <= i; ++j) a[i][j] -= l[i] * col[j];
#pragma unroll
        for (int i = k + 1; i < 6; ++i) a[i][k] = l[i];
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double v = bin[i];
#pragma unroll
        for (int j = 0; j < i; ++j) v -= a[i][j] * y[j];
        y[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) y[i] *= dinv[i];
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        double v = y[i];
#pragma unroll
        for (int j = i + 1; j < 6; ++j) v -= a[j][i] * y[j];
        y[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) x[i] = y[i];
}

KT_HD __forceinline__ void rodrigues_fast(const double* r, double* R)
{
    const double rx = r[0], ry = r[1], rz = r[2];
    const double t2 = rx * rx + ry * ry + rz * rz;
    if (!(t2 <= 0.25)) { rodrigues(r, R); return; }
    // A = sin(t)/t = sum (-1)^k t2^k / (2k+1)!,  B = (1 - cos t)/t^2 = sum (-1)^k t2^k / (2k+2)!
    double A = -1.0 / 121645100408832000.0;        // -1/19!
    double B = -1.0 / 2432902008176640000.0;       // -1/20!
    A = fma(A, t2, 1.0 / 355687428096000.0);   B = fma(B, t2, 1.0 / 6402373705728000.0);      // 17!, 18!
    A = fma(A, t2, -1.0 / 1307674368000.0);    B = fma(B, t2, -1.0 / 20922789888000.0);       // 15!, 16!
    A = fma(A, t2, 1.0 / 6227020800.0);        B = fma(B, t2, 1.0 / 87178291200.0);           // 13!, 14!
    A = fma(A, t2, -1.0 / 39916800.0);         B = fma(B, t2, -1.0 / 479001600.0);            // 11!, 12!
    A = fma(A, t2, 1.0 / 362880.0);            B = fma(B, t2, 1.0 / 3628800.0);               // 9!, 10!
    A = fma(A, t2, -1.0 / 5040.0);             B = fma(B, t2, -1.0 / 40320.0);                // 7!, 8!
    A = fma(A, t2, 1.0 / 120.0);               B = fma(B, t2, 1.0 / 720.0);                   // 5!, 6!
    A = fma(A, t2, -1.0 / 6.0);                B = fma(B, t2, -1.0 / 24.0);                   // 3!, 4!
    A = fma(A, t2, 1.0);                       B = fma(B, t2, 0.5);
    const double c = fma(-t2, B, 1.0);             // cos t
    R[0] = fma(B, rx * rx, c); R[1] = fma(B, rx * ry, -A * rz); R[2] = fma(B, rx * rz, A * ry);
    R[3] = fma(B, rx * ry, A * rz); R[4] = fma(B, ry * ry, c); R[5] = fma(B, ry * rz, -A * rx);
    R[6] = fma(B, rx * rz, -A * ry); R[7] = fma(B, ry * rz, A * rx); R[8] = fma(B, rz * rz, c);
}

KT_HD __forceinline__ void gauss_newton_update_fast(const double* dA, const double* db, double* resultRt,
                                                    const float* Rp, const float* tprev, float* Rcurr, float* tcurr)
{
    double x[6];
    ldlt6_solve_fast(dA, db, x);
    double R[9];
    rodrigues_fast(x + 3, R);
    // resultRt <- [R | x0..2; 0 0 0 1] * resultRt: rows 0..2 only (row 3 of both factors is 0 0 0 1)
    double res[12];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double s = (j == 3) ? x[i] : 0.0;
#pragma unroll
            for (int k = 0; k < 3; ++k) s = fma(R[i * 3 + k], resultRt[k * 4 + j], s);
            res[i * 4 + j] = s;
        }
#pragma unroll
    for (int k = 0; k < 12; ++k) resultRt[k] = res[k];
    float rot[9], tr[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) rot[i * 3 + j] = (float)res[i * 4 + j];
        tr[i] = (float)res[i * 4 + 3];
    }
    float tinv[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) tinv[i] = -dot3_rn(rot[0 * 3 + i], rot[1 * 3 + i], rot[2 * 3 + i], tr[0], tr[1], tr[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j)
            Rcurr[i * 3 + j] = dot3_rn(Rp[i * 3 + 0], Rp[i * 3 + 1], Rp[i * 3 + 2], rot[j * 3 + 0], rot[j * 3 + 1], rot[j * 3 + 2]);
        tcurr[i] = KT_FADD(dot3_rn(Rp[i * 3 + 0], Rp[i * 3 + 1], Rp[i * 3 + 2], tinv[0], tinv[1], tinv[2]), tprev[i]);
    }
}

KT_HD __forceinline__ void gauss_newton_update(const double* dA, const double* db, OdomState* st)
{
    gauss_newton_update_p(dA, db, st->resultRt, st->Rprev, st->tprev, st->Rcurr, st->tcurr);
}

} // namespace kt
