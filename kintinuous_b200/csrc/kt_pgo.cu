// kintinuous_b200 -- pose-graph optimisation on the device: Gauss-Newton over a chain of Pose3d nodes with a prior and loop factors,
// FP64, solved exactly by segment elimination.
//
// Replaces (reference, src/backend/iSAMInterface.cpp, all in iSAM on the CPU there):
//   iSAMInterface::optimise -> isam::Slam::batch_optimization, chi2   :136-140   the Gauss-Newton loop below, pgo_sum_kernel
//   isam::Pose3d_Pose3d_Factor / Pose3d_Factor (slam3d.h, restated)             pgo_linearise_kernel
//   the sparse Cholesky of the normal equations                                 pgo_assemble_kernel .. pgo_backsub_kernel
//
// Residual (iSAM's Pose3d_Pose3d_Factor): e = (p_j (-) p_i).vector() - z over (x, y, z, yaw, pitch, roll), angles wrapped to (-pi, pi],
// whitened by sqrt(1000) (covariance 1e-3 I).  The prior on node 0: e = (Z^-1 p_0).vector() (quirk R4).  Update: t += rho,
// R <- R Exp(phi) per node; with E = T_i^-1 T_j (R_e = R_i^T R_j, t_e = R_i^T (t_j - t_i)) the Jacobians are
//   d t_e / d rho_j = R_i^T,  d t_e / d rho_i = -R_i^T,  d t_e / d phi_i = [t_e]x,
//   d ypr / d phi_j = G(R_e),  d ypr / d phi_i = -G(R_e) R_e^T,   G = [[0, sr/cp, cr/cp], [0, cr, -sr], [1, sr sp/cp, cr sp/cp]]
// (G maps a right perturbation of R_e to yaw / pitch / roll rates; cp = sqrt(R_e[2,1]^2 + R_e[2,2]^2), so a relative pose at pitch
// +-90 degrees gives an infinite G and a failed factorisation, not a wrong step).
//
// Normal equations H d = b: H is block tridiagonal in 6 x 6 blocks (the chain and the prior) plus one off-chain block per loop.  The
// elimination plan (kt_pgo.hpp pgo_plan) cuts each level's chain at every PGO_SEG-th node and at every loop endpoint; one warp per
// segment eliminates its interior by block Cholesky (pgo_segment_kernel) and leaves a 12 x 12 Schur complement on its two separators,
// which form the next level's chain (pgo_gather_kernel).  The last level has no interior; with the loop couplings it is a dense system
// of at most about 6 (2L + 3) unknowns, factorised one block column per launch by a grid of tiles (pgo_dense_panel_kernel) and
// solved by one CTA (pgo_dense_solve_kernel).  Back-substitution runs down the levels, one thread per segment.
//
// Determinism: no floating-point atomics; every sum has a fixed order; every output element has one writer.  Two runs give the same bits.
#include "kt_ops.h"
#include "kt_pgo.hpp"
#include "../../include/kintinuous_b200.h"
#include <vector>
#include <cmath>
#include <cstring>

namespace kt {

namespace {

const int LIN_THREADS = 128;
const int SUM_THREADS = 1024;
const int TILE = 32;
const int SOLVE_THREADS = 512;
const double WHITEN = 31.622776601683793;       // sqrt(1 / 1e-3)

struct Rt { double R[9]; double t[3]; };

__device__ __forceinline__ Rt load_pose(const double* X)
{
    Rt p;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) p.R[3 * r + c] = X[4 * r + c];
        p.t[r] = X[4 * r + 3];
    }
    return p;
}

__device__ __forceinline__ double wrap_angle(double a)
{
    double r = fmod(a + M_PI, 2.0 * M_PI);
    if (r <= 0.0) r += 2.0 * M_PI;
    return r - M_PI;
}

__device__ __forceinline__ Rt pose_of_vector(const double* v)
{
    Rt p;
    const double cy = cos(v[3]), sy = sin(v[3]), cp = cos(v[4]), sp = sin(v[4]), cr = cos(v[5]), sr = sin(v[5]);
    p.R[0] = cy * cp; p.R[1] = cy * sp * sr - sy * cr; p.R[2] = cy * sp * cr + sy * sr;
    p.R[3] = sy * cp; p.R[4] = sy * sp * sr + cy * cr; p.R[5] = sy * sp * cr - cy * sr;
    p.R[6] = -sp;     p.R[7] = cp * sr;                p.R[8] = cp * cr;
    p.t[0] = v[0]; p.t[1] = v[1]; p.t[2] = v[2];
    return p;
}

// ---- linearisation: one thread per factor --------------------------------------------------------------------------------------
// Writes the whitened error (6), J_i and J_j (6 x 6 row-major, columns rho then phi; J_i is zero for the prior) and |e|^2.
__global__ void __launch_bounds__(LIN_THREADS)
pgo_linearise_kernel(const double* __restrict__ X, const PgoFactor* __restrict__ f, int nf,
                     double* __restrict__ E, double* __restrict__ JI, double* __restrict__ JJ, double* __restrict__ e2)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nf) return;
    const PgoFactor F = f[k];
    const bool prior = F.i < 0;
    const Rt pi = prior ? pose_of_vector(F.z) : load_pose(X + 16 * F.i);
    const Rt pj = load_pose(X + 16 * F.j);
    double Re[9], te[3];
    const double dt[3] = {pj.t[0] - pi.t[0], pj.t[1] - pi.t[1], pj.t[2] - pi.t[2]};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) Re[3 * r + c] = pi.R[r] * pj.R[c] + pi.R[3 + r] * pj.R[3 + c] + pi.R[6 + r] * pj.R[6 + c];
        te[r] = pi.R[r] * dt[0] + pi.R[3 + r] * dt[1] + pi.R[6 + r] * dt[2];
    }
    const double cp = sqrt(Re[7] * Re[7] + Re[8] * Re[8]);
    const double yaw = atan2(Re[3], Re[0]), pitch = atan2(-Re[6], cp), roll = atan2(Re[7], Re[8]);
    double e[6];
    if (prior) {
        e[0] = te[0]; e[1] = te[1]; e[2] = te[2];
        e[3] = wrap_angle(yaw); e[4] = wrap_angle(pitch); e[5] = wrap_angle(roll);
    } else {
        e[0] = te[0] - F.z[0]; e[1] = te[1] - F.z[1]; e[2] = te[2] - F.z[2];
        e[3] = wrap_angle(yaw - F.z[3]); e[4] = wrap_angle(pitch - F.z[4]); e[5] = wrap_angle(roll - F.z[5]);
    }
    double sq = 0.0;
#pragma unroll
    for (int q = 0; q < 6; ++q) { e[q] *= WHITEN; E[6 * k + q] = e[q]; sq += e[q] * e[q]; }
    e2[k] = sq;
    const double sr = sin(roll), cr = cos(roll), sp = -Re[6];
    const double G[9] = {0.0, sr / cp, cr / cp, 0.0, cr, -sr, 1.0, sr * sp / cp, cr * sp / cp};
    double* jj = JJ + 36 * (size_t)k;
    double* ji = JI + 36 * (size_t)k;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            jj[6 * r + c] = WHITEN * pi.R[3 * c + r];               // R_i^T
            jj[6 * r + 3 + c] = 0.0;
            jj[6 * (3 + r) + c] = 0.0;
            jj[6 * (3 + r) + 3 + c] = WHITEN * G[3 * r + c];
            ji[6 * r + c] = -WHITEN * pi.R[3 * c + r];
            ji[6 * (3 + r) + c] = 0.0;
            // -G R_e^T
            ji[6 * (3 + r) + 3 + c] = -WHITEN * (G[3 * r] * Re[3 * c] + G[3 * r + 1] * Re[3 * c + 1] + G[3 * r + 2] * Re[3 * c + 2]);
        }
    }
    // [t_e]x
    ji[3] = 0.0;               ji[4] = -WHITEN * te[2];  ji[5] = WHITEN * te[1];
    ji[9] = WHITEN * te[2];    ji[10] = 0.0;             ji[11] = -WHITEN * te[0];
    ji[15] = -WHITEN * te[1];  ji[16] = WHITEN * te[0];  ji[17] = 0.0;
}

// Fixed-order sum of n doubles (one CTA): thread t adds t, t + T, ... in order, then a tree.  out[0] = the sum.
__global__ void __launch_bounds__(SUM_THREADS)
pgo_sum_kernel(const double* __restrict__ v, int n, double* __restrict__ out)
{
    __shared__ double red[SUM_THREADS];
    double s = 0.0;
    for (int k = threadIdx.x; k < n; k += SUM_THREADS) s += v[k];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = SUM_THREADS / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = red[0];
}

// acc(r, c) += sum_m A(m, r) B(m, c) for 6 x 6 row-major A, B (A^T B)
__device__ __forceinline__ double atb(const double* A, const double* B, int r, int c)
{
    double s = 0.0;
#pragma unroll
    for (int m = 0; m < 6; ++m) s += A[6 * m + r] * B[6 * m + c];
    return s;
}
__device__ __forceinline__ double atv(const double* A, const double* v, int r)
{
    double s = 0.0;
#pragma unroll
    for (int m = 0; m < 6; ++m) s += A[6 * m + r] * v[m];
    return s;
}

// ---- normal equations: one thread per node, plus one per loop for its off-chain block ---------------------------------------
// Node k gathers, in this order, the prior (k = 0), odometry factor k (as j), odometry factor k + 1 (as i) and its loop factors
// (CSR, ascending).  D[k] = H(k, k), C[k] = H(k, k - 1), b[k] = -(J^T e)_k.  Thread n + l writes HL[l] = H(j_l, i_l).
__global__ void __launch_bounds__(128)
pgo_assemble_kernel(int n, int nf, const PgoFactor* __restrict__ f, const double* __restrict__ E, const double* __restrict__ JI,
                    const double* __restrict__ JJ, const int* __restrict__ loff, const int* __restrict__ lidx,
                    double* __restrict__ D, double* __restrict__ C, double* __restrict__ b, double* __restrict__ HL)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nf) return;
    if (k >= n) {
        const int l = k - n, fi = n + l;
        for (int q = 0; q < 36; ++q) HL[36 * l + q] = atb(JJ + 36 * (size_t)fi, JI + 36 * (size_t)fi, q / 6, q % 6);
        return;
    }
    for (int q = 0; q < 42; ++q) {
        const int r = q < 36 ? q / 6 : q - 36, c = q % 6;
        double s = 0.0;
        auto add = [&](const double* J, const double* e) { s += q < 36 ? atb(J, J, r, c) : -atv(J, e, r); };
        if (k == 0) add(JJ, E);
        if (k >= 1) add(JJ + 36 * (size_t)k, E + 6 * (size_t)k);
        if (k + 1 < n) add(JI + 36 * (size_t)(k + 1), E + 6 * (size_t)(k + 1));
        for (int p = loff[k]; p < loff[k + 1]; ++p) {
            const int fi = lidx[p];
            add(f[fi].i == k ? JI + 36 * (size_t)fi : JJ + 36 * (size_t)fi, E + 6 * (size_t)fi);
        }
        if (q < 36) D[36 * (size_t)k + q] = s; else b[6 * (size_t)k + r] = s;
    }
    for (int q = 0; q < 36; ++q)
        C[36 * (size_t)k + q] = k >= 1 ? atb(JJ + 36 * (size_t)k, JI + 36 * (size_t)k, q / 6, q % 6) : 0.0;
}

// ---- segment elimination: one warp per segment ----------------------------------------------------------------------------------
// 6 x 6 Cholesky of S (row-major, lower part used) into L by one thread; false on a pivot that is not positive or not finite.
__device__ bool chol6(const double* S, double* L)
{
    for (int q = 0; q < 36; ++q) L[q] = 0.0;
    for (int c = 0; c < 6; ++c) {
        double d = S[6 * c + c];
        for (int m = 0; m < c; ++m) d -= L[6 * c + m] * L[6 * c + m];
        if (!(d > 0.0) || !isfinite(d)) return false;
        const double l = sqrt(d);
        L[6 * c + c] = l;
        for (int r = c + 1; r < 6; ++r) {
            double v = S[6 * r + c];
            for (int m = 0; m < c; ++m) v -= L[6 * r + m] * L[6 * c + m];
            L[6 * r + c] = v / l;
        }
    }
    return true;
}
// column col of L^-1 B (B row-major 6 x 6, or B^T when trans) into out (row-major)
__device__ __forceinline__ void lsolve_col(const double* L, const double* B, bool trans, int col, double* out)
{
    double y[6];
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        double v = trans ? B[6 * col + r] : B[6 * r + col];
#pragma unroll
        for (int m = 0; m < r; ++m) v -= L[6 * r + m] * y[m];
        y[r] = v / L[6 * r + r];
    }
#pragma unroll
    for (int r = 0; r < 6; ++r) out[6 * r + col] = y[r];
}
__device__ __forceinline__ void lsolve_vec(const double* L, const double* g, double* out)
{
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        double v = g[r];
#pragma unroll
        for (int m = 0; m < r; ++m) v -= L[6 * r + m] * out[m];
        out[r] = v / L[6 * r + r];
    }
}

// Segment s of a level: separators a = sep[s], b = sep[s + 1], interior a + 1 .. b - 1.  For each interior node in turn (D' its
// current diagonal, A' its current coupling to a, g' its current right-hand side): L = chol(D'), W = L^-1 A', w = L^-1 g',
// V = L^-1 C[k+1]^T; a gains -W^T W and -W^T w; the next node's D' = D - V^T V, A' = -V^T W, g' = g - V^T w.  L, A', g' are kept in
// D, A, g for the back-substitution.  Out per segment: Saa, Sbb (to subtract from the separators' diagonals), Sba = H'(b, a), ga, gb.
__global__ void __launch_bounds__(32)
pgo_segment_kernel(const int* __restrict__ sep, double* __restrict__ D, const double* __restrict__ C, double* __restrict__ g,
                   double* __restrict__ A, double* __restrict__ Saa, double* __restrict__ Sbb, double* __restrict__ Sba,
                   double* __restrict__ ga, double* __restrict__ gb, int* __restrict__ fail)
{
    __shared__ double Dc[36], Ac[36], gc[6], L[36], W[36], V[36], w[6], Sa[36], sa[6], Dn[36], An[36], gn[6];
    __shared__ int bad;
    const int s = blockIdx.x, lane = threadIdx.x;
    const int a = sep[s], b = sep[s + 1];
    double* saa = Saa + 36 * (size_t)s; double* sbb = Sbb + 36 * (size_t)s; double* sba = Sba + 36 * (size_t)s;
    if (b == a + 1) {
        for (int q = lane; q < 36; q += 32) { saa[q] = 0.0; sbb[q] = 0.0; sba[q] = C[36 * (size_t)b + q]; }
        if (lane < 6) { ga[6 * s + lane] = 0.0; gb[6 * s + lane] = 0.0; }
        return;
    }
    for (int q = lane; q < 36; q += 32) { Dc[q] = D[36 * (size_t)(a + 1) + q]; Ac[q] = C[36 * (size_t)(a + 1) + q]; Sa[q] = 0.0; }
    if (lane < 6) { gc[lane] = g[6 * (size_t)(a + 1) + lane]; sa[lane] = 0.0; }
    if (lane == 0) bad = 0;
    __syncthreads();
    for (int k = a + 1; k < b; ++k) {
        if (lane == 0 && !chol6(Dc, L)) { bad = 1; *fail = 1; }
        __syncthreads();
        if (bad) return;
        for (int q = lane; q < 36; q += 32) { D[36 * (size_t)k + q] = L[q]; A[36 * (size_t)k + q] = Ac[q]; }
        if (lane < 6) g[6 * (size_t)k + lane] = gc[lane];
        const double* Bn = C + 36 * (size_t)(k + 1);             // H(k + 1, k)
        if (lane < 6) lsolve_col(L, Ac, false, lane, W);
        else if (lane < 12) lsolve_col(L, Bn, true, lane - 6, V);
        else if (lane == 12) lsolve_vec(L, gc, w);
        __syncthreads();
        const bool last = k + 1 == b;
        for (int q = lane; q < 36; q += 32) {
            const int r = q / 6, c = q % 6;
            Sa[q] += atb(W, W, r, c);
            const double vv = atb(V, V, r, c), vw = atb(V, W, r, c);
            Dn[q] = last ? vv : D[36 * (size_t)(k + 1) + q] - vv;
            An[q] = -vw;
        }
        if (lane < 6) {
            sa[lane] += atv(W, w, lane);
            const double vg = atv(V, w, lane);
            gn[lane] = last ? vg : g[6 * (size_t)(k + 1) + lane] - vg;
        }
        __syncthreads();
        for (int q = lane; q < 36; q += 32) { Dc[q] = Dn[q]; Ac[q] = An[q]; }
        if (lane < 6) gc[lane] = gn[lane];
        __syncthreads();
    }
    for (int q = lane; q < 36; q += 32) { saa[q] = Sa[q]; sbb[q] = Dc[q]; sba[q] = Ac[q]; }
    if (lane < 6) { ga[6 * s + lane] = sa[lane]; gb[6 * s + lane] = gc[lane]; }
}

// The next level's chain: node p is separator sep[p]; one thread per (node, entry)
__global__ void pgo_gather_kernel(int P, const int* __restrict__ sep, const double* __restrict__ D, const double* __restrict__ g,
                                  const double* __restrict__ Saa, const double* __restrict__ Sbb, const double* __restrict__ Sba,
                                  const double* __restrict__ ga, const double* __restrict__ gb,
                                  double* __restrict__ D1, double* __restrict__ C1, double* __restrict__ g1)
{
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)P * 42) return;
    const int p = (int)(t / 42), q = (int)(t % 42);
    const int k = sep[p];
    if (q < 36) {
        double v = D[36 * (size_t)k + q];
        if (p + 1 < P) v -= Saa[36 * (size_t)p + q];
        if (p > 0) v -= Sbb[36 * (size_t)(p - 1) + q];
        D1[36 * (size_t)p + q] = v;
        C1[36 * (size_t)p + q] = p > 0 ? Sba[36 * (size_t)(p - 1) + q] : 0.0;
    } else {
        const int r = q - 36;
        double v = g[6 * (size_t)k + r];
        if (p + 1 < P) v -= ga[6 * (size_t)p + r];
        if (p > 0) v -= gb[6 * (size_t)(p - 1) + r];
        g1[6 * (size_t)p + r] = v;
    }
}

// ---- the top level: dense ---------------------------------------------------------------------------------------------------
// M (N x N, N = 6K, row-major) from the chain blocks; the loop blocks are added by pgo_dense_loops_kernel, one loop after another.
__global__ void pgo_dense_fill_kernel(int K, const double* __restrict__ D, const double* __restrict__ C, double* __restrict__ M)
{
    const int N = 6 * K;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)N * N) return;
    const int r = (int)(t / N), c = (int)(t % N), p = r / 6, q = c / 6;
    double v = 0.0;
    if (p == q) v = D[36 * (size_t)p + 6 * (r % 6) + c % 6];
    else if (p == q + 1) v = C[36 * (size_t)p + 6 * (r % 6) + c % 6];
    else if (q == p + 1) v = C[36 * (size_t)q + 6 * (c % 6) + r % 6];
    M[t] = v;
}
__global__ void pgo_dense_loops_kernel(int K, int L, const int* __restrict__ ti, const int* __restrict__ tj, const double* __restrict__ HL,
                                       double* __restrict__ M)
{
    const int N = 6 * K, q = threadIdx.x;
    for (int l = 0; l < L; ++l) {
        if (q < 36) {
            const int r = q / 6, c = q % 6;
            const double h = HL[36 * l + q];                   // H(j, i)(r, c)
            M[(size_t)(6 * tj[l] + r) * N + 6 * ti[l] + c] += h;
            M[(size_t)(6 * ti[l] + c) * N + 6 * tj[l] + r] += h;
        }
        __syncthreads();
    }
}

// Block column j0 .. j0 + 5 of the right-looking Cholesky: every CTA factorises the 6 x 6 diagonal block of M (the same bits in all),
// forms the panel rows L(i, j0..) = M(i, j0..) L_jj^-T its tile needs, and updates its TILE x TILE tile of the trailing lower
// triangle of M.  CTAs of tile column 0 write their rows of the panel (and CTA 0 the diagonal block) into Lf, a separate array,
// so that no CTA reads what another writes.
__global__ void __launch_bounds__(TILE * 8)
pgo_dense_panel_kernel(int N, int j0, double* __restrict__ M, double* __restrict__ Lf, int* __restrict__ fail)
{
    __shared__ double Sd[36], Ld[36], Pr[TILE][6], Pc[TILE][6];
    __shared__ int ok;
    if (*fail) return;
    const int tid = threadIdx.x;
    // tile (ti, tk), tk <= ti, of the trailing matrix starting at j0 + 6
    int ti = 0, rem = blockIdx.x;
    while (rem > ti) { rem -= ti + 1; ++ti; }
    const int tk = rem;
    const int base = j0 + 6;
    if (tid < 36) Sd[tid] = M[(size_t)(j0 + tid / 6) * N + j0 + tid % 6];
    __syncthreads();
    if (tid == 0) {
        ok = chol6(Sd, Ld);
        if (!ok) *fail = 1;
    }
    __syncthreads();
    if (!ok) return;
    if (blockIdx.x == 0 && tid < 36) Lf[(size_t)(j0 + tid / 6) * N + j0 + tid % 6] = Ld[tid];
    for (int u = tid; u < 2 * TILE; u += blockDim.x) {
        const int i = base + (u < TILE ? ti * TILE + u : tk * TILE + u - TILE);
        double* dst = u < TILE ? &Pr[u][0] : &Pc[u - TILE][0];
        if (i >= N) { for (int c = 0; c < 6; ++c) dst[c] = 0.0; continue; }
        const double* row = M + (size_t)i * N + j0;
        for (int c = 0; c < 6; ++c) {
            double v = row[c];
            for (int m = 0; m < c; ++m) v -= dst[m] * Ld[6 * c + m];
            dst[c] = v / Ld[6 * c + c];
        }
        if (u < TILE && tk == 0) for (int c = 0; c < 6; ++c) Lf[(size_t)i * N + j0 + c] = dst[c];
    }
    __syncthreads();
    for (int u = tid; u < TILE * TILE; u += blockDim.x) {
        const int r = u / TILE, c = u % TILE;
        const int i = base + ti * TILE + r, k = base + tk * TILE + c;
        if (i >= N || k > i) continue;
        double s = 0.0;
#pragma unroll
        for (int m = 0; m < 6; ++m) s += Pr[r][m] * Pc[c][m];
        M[(size_t)i * N + k] -= s;
    }
}

// Lf y = rhs, Lf^T x = y, one CTA, 6 x 6 blocks: the diagonal block by one thread, the rest of the column by all
__global__ void __launch_bounds__(SOLVE_THREADS)
pgo_dense_solve_kernel(int N, const double* __restrict__ Lf, double* __restrict__ v, const int* __restrict__ fail)
{
    if (*fail) return;
    const int tid = threadIdx.x;
    for (int j0 = 0; j0 < N; j0 += 6) {
        if (tid == 0)
            for (int r = j0; r < j0 + 6; ++r) {
                double s = v[r];
                for (int m = j0; m < r; ++m) s -= Lf[(size_t)r * N + m] * v[m];
                v[r] = s / Lf[(size_t)r * N + r];
            }
        __syncthreads();
        for (int i = j0 + 6 + tid; i < N; i += SOLVE_THREADS) {
            double s = 0.0;
            for (int m = j0; m < j0 + 6; ++m) s += Lf[(size_t)i * N + m] * v[m];
            v[i] -= s;
        }
        __syncthreads();
    }
    for (int j0 = N - 6; j0 >= 0; j0 -= 6) {
        if (tid == 0)
            for (int r = j0 + 5; r >= j0; --r) {
                double s = v[r];
                for (int m = r + 1; m < j0 + 6; ++m) s -= Lf[(size_t)m * N + r] * v[m];
                v[r] = s / Lf[(size_t)r * N + r];
            }
        __syncthreads();
        for (int i = tid; i < j0; i += SOLVE_THREADS) {
            double s = 0.0;
            for (int m = j0; m < j0 + 6; ++m) s += Lf[(size_t)m * N + i] * v[m];
            v[i] -= s;
        }
        __syncthreads();
    }
}

// ---- back-substitution: one thread per segment ---------------------------------------------------------------------------------
// x of level l from x1 of level l + 1: the separators copy, the interior k = b - 1 .. a + 1 solve
// L L^T x_k = g'_k - A'_k x_a - C[k + 1]^T x_{k+1}.
__global__ void pgo_backsub_kernel(int S, const int* __restrict__ sep, const double* __restrict__ Lk, const double* __restrict__ A,
                                   const double* __restrict__ C, const double* __restrict__ g, const double* __restrict__ x1,
                                   double* __restrict__ x, const int* __restrict__ fail)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || *fail) return;
    const int a = sep[s], b = sep[s + 1];
    double xa[6], xn[6];
    for (int r = 0; r < 6; ++r) { xa[r] = x1[6 * s + r]; xn[r] = x1[6 * (s + 1) + r]; x[6 * (size_t)a + r] = xa[r]; }
    if (s == S - 1) for (int r = 0; r < 6; ++r) x[6 * (size_t)b + r] = xn[r];
    for (int k = b - 1; k > a; --k) {
        const double* L = Lk + 36 * (size_t)k; const double* Ak = A + 36 * (size_t)k; const double* Cn = C + 36 * (size_t)(k + 1);
        double rhs[6], y[6];
        for (int r = 0; r < 6; ++r) {
            double v = g[6 * (size_t)k + r];
            for (int m = 0; m < 6; ++m) v -= Ak[6 * r + m] * xa[m] + Cn[6 * m + r] * xn[m];
            rhs[r] = v;
        }
        for (int r = 0; r < 6; ++r) { double v = rhs[r]; for (int m = 0; m < r; ++m) v -= L[6 * r + m] * y[m]; y[r] = v / L[6 * r + r]; }
        for (int r = 5; r >= 0; --r) { double v = y[r]; for (int m = r + 1; m < 6; ++m) v -= L[6 * m + r] * xn[m]; xn[r] = v / L[6 * r + r]; }
        for (int r = 0; r < 6; ++r) x[6 * (size_t)k + r] = xn[r];
    }
}

// t += rho, R <- R Exp(phi); nothing when the factorisation failed
__global__ void pgo_update_kernel(int n, const double* __restrict__ dx, double* __restrict__ X, const int* __restrict__ fail)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n || *fail) return;
    const double* d = dx + 6 * (size_t)k;
    double* P = X + 16 * (size_t)k;
    const double th2 = d[3] * d[3] + d[4] * d[4] + d[5] * d[5], th = sqrt(th2);
    double sa, sb;                                                  // sin(th) / th, (1 - cos(th)) / th^2
    if (th < 1e-8) { sa = 1.0; sb = 0.5; } else { sa = sin(th) / th; sb = (1.0 - cos(th)) / th2; }
    const double wx = d[3], wy = d[4], wz = d[5];
    const double E[9] = {1.0 - sb * (wy * wy + wz * wz), -sa * wz + sb * wx * wy, sa * wy + sb * wx * wz,
                         sa * wz + sb * wx * wy, 1.0 - sb * (wx * wx + wz * wz), -sa * wx + sb * wy * wz,
                         -sa * wy + sb * wx * wz, sa * wx + sb * wy * wz, 1.0 - sb * (wx * wx + wy * wy)};
    double R[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) R[3 * r + c] = P[4 * r] * E[c] + P[4 * r + 1] * E[3 + c] + P[4 * r + 2] * E[6 + c];
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) P[4 * r + c] = R[3 * r + c]; P[4 * r + 3] += d[r]; }
}

template <class T> int dalloc(std::vector<void*>& owned, T** p, size_t count)
{
    void* q = 0;
    KT_CUDA(cudaMalloc(&q, (count ? count : 1) * sizeof(T)));
    owned.push_back(q); *p = (T*)q;
    return 0;
}

} // namespace

int pgo_optimise(const double* poses_in, int n, const PgoFactor* fh, int nf, double* X, kt_pgo_report* rep, cudaStream_t s)
{
    std::memset(rep, 0, sizeof(*rep));
    rep->nodes = n; rep->factors = nf; rep->loops = nf - n;
    if (n > PGO_MAX_NODES) { set_error("pgo_optimise: %d nodes, at most %d", n, PGO_MAX_NODES); return KT_ERR_CAPACITY; }
    const int chk = pgo_check_factors(fh, nf, n);
    if (chk) { set_error("pgo_optimise: the factor list is not a prior on node 0, the chain 0 -> 1 -> ... -> %d and loops (check %d)", n - 1, chk); return KT_ERR_INVALID; }
    const int L = nf - n;
    if (L > PGO_MAX_LOOPS) { set_error("pgo_optimise: %d loop factors, at most %d", L, PGO_MAX_LOOPS); return KT_ERR_CAPACITY; }
    std::vector<int> li(L), lj(L);
    for (int l = 0; l < L; ++l) { li[l] = fh[n + l].i; lj[l] = fh[n + l].j; }
    const PgoPlan plan = pgo_plan(n, li, lj);
    const int top = plan.top(), K = plan.n[top], N = 6 * K;
    std::vector<int> loff, lidx; pgo_loop_csr(fh, nf, n, loff, lidx);

    std::vector<void*> owned;
    cudaEvent_t ev[2] = {0, 0};
    auto run = [&]() -> int {
        PgoFactor* d_f; double *d_E, *d_JI, *d_JJ, *d_e2, *d_HL, *d_out, *d_M, *d_Lf; int *d_loff, *d_lidx, *d_fail, *d_ti, *d_tj;
        if (dalloc(owned, &d_f, nf) || dalloc(owned, &d_E, 6 * (size_t)nf) || dalloc(owned, &d_JI, 36 * (size_t)nf) || dalloc(owned, &d_JJ, 36 * (size_t)nf) ||
            dalloc(owned, &d_e2, nf) || dalloc(owned, &d_HL, 36 * (size_t)(L ? L : 1)) || dalloc(owned, &d_out, 2) || dalloc(owned, &d_M, (size_t)N * N) ||
            dalloc(owned, &d_Lf, (size_t)N * N) || dalloc(owned, &d_loff, n + 1) || dalloc(owned, &d_lidx, lidx.size()) || dalloc(owned, &d_fail, 1) ||
            dalloc(owned, &d_ti, L) || dalloc(owned, &d_tj, L)) return KT_ERR_CUDA;
        // per level: D, C, g, A, x; per level below the top: sep and the segment outputs
        std::vector<double*> D(top + 1), C(top + 1), g(top + 1), A(top + 1), x(top + 1);
        std::vector<int*> sep(top);
        std::vector<double*> Saa(top), Sbb(top), Sba(top), ga(top), gb(top);
        for (int l = 0; l <= top; ++l) {
            const size_t m = plan.n[l];
            if (dalloc(owned, &D[l], 36 * m) || dalloc(owned, &C[l], 36 * m) || dalloc(owned, &g[l], 6 * m) || dalloc(owned, &A[l], 36 * m) || dalloc(owned, &x[l], 6 * m)) return KT_ERR_CUDA;
            if (l < top) {
                const size_t S = plan.sep[l].size() - 1;
                if (dalloc(owned, &sep[l], S + 1) || dalloc(owned, &Saa[l], 36 * S) || dalloc(owned, &Sbb[l], 36 * S) || dalloc(owned, &Sba[l], 36 * S) ||
                    dalloc(owned, &ga[l], 6 * S) || dalloc(owned, &gb[l], 6 * S)) return KT_ERR_CUDA;
                KT_CUDA(cudaMemcpyAsync(sep[l], plan.sep[l].data(), (S + 1) * sizeof(int), cudaMemcpyHostToDevice, s));
            }
        }
        KT_CUDA(cudaMemcpyAsync(d_f, fh, nf * sizeof(PgoFactor), cudaMemcpyHostToDevice, s));
        KT_CUDA(cudaMemcpyAsync(d_loff, loff.data(), loff.size() * sizeof(int), cudaMemcpyHostToDevice, s));
        if (!lidx.empty()) KT_CUDA(cudaMemcpyAsync(d_lidx, lidx.data(), lidx.size() * sizeof(int), cudaMemcpyHostToDevice, s));
        if (L) {
            KT_CUDA(cudaMemcpyAsync(d_ti, plan.loop_i.data(), L * sizeof(int), cudaMemcpyHostToDevice, s));
            KT_CUDA(cudaMemcpyAsync(d_tj, plan.loop_j.data(), L * sizeof(int), cudaMemcpyHostToDevice, s));
        }
        if (X != poses_in) KT_CUDA(cudaMemcpyAsync(X, poses_in, 16 * (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
        KT_CUDA(cudaMemsetAsync(d_fail, 0, sizeof(int), s));
        // chi2 and the failure flag of the current poses: the one read-back of a step.  `done` (optional) is recorded after the sum.
        double chi2 = 0.0; int failed = 0;
        auto linearise = [&](cudaEvent_t done) -> int {
            pgo_linearise_kernel<<<(nf + LIN_THREADS - 1) / LIN_THREADS, LIN_THREADS, 0, s>>>(X, d_f, nf, d_E, d_JI, d_JJ, d_e2); KT_LAUNCH_CHECK();
            pgo_sum_kernel<<<1, SUM_THREADS, 0, s>>>(d_e2, nf, d_out); KT_LAUNCH_CHECK();
            if (done) KT_CUDA(cudaEventRecord(done, s));
            KT_CUDA(cudaMemcpyAsync(&chi2, d_out, sizeof(double), cudaMemcpyDeviceToHost, s));
            KT_CUDA(cudaMemcpyAsync(&failed, d_fail, sizeof(int), cudaMemcpyDeviceToHost, s));
            KT_CUDA(cudaStreamSynchronize(s));
            return 0;
        };
        // device time of each step, from the assembly to the chi2 of the updated poses (kt_pgo_report::step_ms)
        KT_CUDA(cudaEventCreate(&ev[0])); KT_CUDA(cudaEventCreate(&ev[1]));
        int r = linearise(0); if (r) return r;
        double prev = chi2, step_ms = 0.0;
        rep->chi2_initial = rep->chi2_final = prev;
        for (int it = 0; it < 100; ++it) {
            KT_CUDA(cudaEventRecord(ev[0], s));
            pgo_assemble_kernel<<<(nf + 127) / 128, 128, 0, s>>>(n, nf, d_f, d_E, d_JI, d_JJ, d_loff, d_lidx, D[0], C[0], g[0], d_HL); KT_LAUNCH_CHECK();
            for (int l = 0; l < top; ++l) {
                const int S = (int)plan.sep[l].size() - 1, P = plan.n[l + 1];
                pgo_segment_kernel<<<S, 32, 0, s>>>(sep[l], D[l], C[l], g[l], A[l], Saa[l], Sbb[l], Sba[l], ga[l], gb[l], d_fail); KT_LAUNCH_CHECK();
                pgo_gather_kernel<<<(unsigned)(((size_t)P * 42 + 255) / 256), 256, 0, s>>>(P, sep[l], D[l], g[l], Saa[l], Sbb[l], Sba[l], ga[l], gb[l],
                                                                                              D[l + 1], C[l + 1], g[l + 1]); KT_LAUNCH_CHECK();
            }
            pgo_dense_fill_kernel<<<(unsigned)(((size_t)N * N + 255) / 256), 256, 0, s>>>(K, D[top], C[top], d_M); KT_LAUNCH_CHECK();
            if (L) { pgo_dense_loops_kernel<<<1, 64, 0, s>>>(K, L, d_ti, d_tj, d_HL, d_M); KT_LAUNCH_CHECK(); }
            for (int j0 = 0; j0 < N; j0 += 6) {
                const int T = (N - j0 - 6 + TILE - 1) / TILE, tiles = T > 0 ? T * (T + 1) / 2 : 1;
                pgo_dense_panel_kernel<<<tiles, TILE * 8, 0, s>>>(N, j0, d_M, d_Lf, d_fail); KT_LAUNCH_CHECK();
            }
            KT_CUDA(cudaMemcpyAsync(x[top], g[top], (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, s));
            pgo_dense_solve_kernel<<<1, SOLVE_THREADS, 0, s>>>(N, d_Lf, x[top], d_fail); KT_LAUNCH_CHECK();
            for (int l = top - 1; l >= 0; --l) {
                const int S = (int)plan.sep[l].size() - 1;
                pgo_backsub_kernel<<<(S + 127) / 128, 128, 0, s>>>(S, sep[l], D[l], A[l], C[l], g[l], x[l + 1], x[l], d_fail); KT_LAUNCH_CHECK();
            }
            pgo_update_kernel<<<(n + 127) / 128, 128, 0, s>>>(n, x[0], X, d_fail); KT_LAUNCH_CHECK();
            r = linearise(ev[1]); if (r) return r;
            float ms = 0.f;
            KT_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
            step_ms += ms;
            rep->iterations = it + 1;
            rep->step_ms = step_ms / rep->iterations;
            if (failed) { rep->solver_failed = 1; break; }
            const double dec = prev - chi2;
            rep->chi2_final = chi2;
            if (dec < 1e-3 || dec < 1e-5 * prev) break;
            prev = chi2;
        }
        return 0;
    };
    const int r = run();
    cudaStreamSynchronize(s);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    for (void* p : owned) cudaFree(p);
    return r;
}

} // namespace kt
