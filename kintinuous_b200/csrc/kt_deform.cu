// kintinuous_b200 -- the embedded deformation graph on the device: vertex weights, Gauss-Newton normal equations, a block-banded FP64
// Cholesky solve and the map update.
//
// Replaces (reference, src/backend/DeformationGraph.cpp, all on the CPU there):
//   weightVerticesSeq                          :441-556   deform_weight_kernel
//   optimiseGraphSparse / sparseResidual(Cons)  :714-774, :930-988, DeformationGraph.h:261-281   deform_residual_kernel + host loop
//   sparseJacobian + CholeskyDecomp::solve      :776-928 (CHOLMOD)                              deform_assemble_kernel + deform_solve_kernel
//   applyDeltaSparse                           :999-1026  inside deform_solve_kernel
//   applyGraphToVertices / computeVertexPosition :644-677, :1028-1054 (8 boost threads)         deform_apply_kernel
//
// Unknowns: 12 per node, the rotation in Eigen's column-major order (x[3m+e] = R(e,m)) then the translation.  Every term of the cost
// except E_rot is affine in the unknowns with a constant Jacobian, r_e = sum over its nodes j, m = 0..3 of u_j[m] x_j[3m+e] + c_e:
//   E_reg (edge j -> n, weight 10):   u_j = s (g_n - g_j, 1), u_n = s (0, 0, 0, -1), c = s (g_j - g_n)            s = sqrt(10)
//   E_con (vertex v, weights w_j):    u_j = s w_j (v - g_j, 1),                      c = s (sum_j w_j g_j - target)  s = 10
// so its block of J^T J between nodes a and b is (u_a u_b^T) (x) I_3, which is how deform_assemble_kernel builds the band.  A vertex's
// nodes lie in a window of 20 consecutive nodes and edges join nodes at most k apart, so J^T J has 12 x 12 blocks only within
// DEFORM_BAND = 19 blocks of the diagonal; the host checks that bound while it builds the terms.
//
// Determinism: no floating-point atomics.  Every entry of the band and of the right-hand side is the sum of its terms in a fixed order
// (node-major lists built on the host), the factorisation runs in one CTA with a fixed assignment of entries to threads, and the
// norms are fixed-order block reductions.  Two runs give the same bits.
#include "kt_ops.h"
#include "kt_deform.hpp"
#include "../../include/kintinuous_b200.h"
#include <vector>
#include <cmath>
#include <cstring>
#include <algorithm>
#include <climits>

namespace kt {

namespace {

const int DK = DEFORM_K;
const int BW = DEFORM_BAND + 1;                  // blocks stored per block row: (i, i), (i, i-1), ..., (i, i-19)
const int SOLVE_THREADS = 512;
const int RES_THREADS = 512;
const int ASM_THREADS = BW * 16;                 // one thread per (block, m, m') of the 4 x 4 kernel of a block

// ---- weights (weightVerticesSeq :450-555) ----------------------------------------------------------------------------------
// One thread per vertex.  The candidate distances are float, as the reference's getVector3fMap().norm(), with no FMA contraction
// and a correctly rounded sqrt; the k + 1 nearest are kept ordered by (distance, node id) -- std::sort leaves ties unordered, this
// breaks them by id.  The weights are FP64: (1 - |v - g_j| / dMax)^2 for the k nearest, normalised, then sorted by node id.
__global__ void __launch_bounds__(256)
deform_weight_kernel(const float* __restrict__ node_pos, const uint64_t* __restrict__ node_times, int n_nodes,
                     const unsigned char* __restrict__ pts, size_t stride, const uint64_t* __restrict__ times, size_t n,
                     int4* __restrict__ ids, double* __restrict__ weights)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* p = (const float*)(pts + i * stride);
    const float vx = p[0], vy = p[1], vz = p[2];
    const int found = deform_nearest_node(node_times, n_nodes, times[i]);
    int lo, hi; deform_window(found, n_nodes, &lo, &hi);
    float bd[DK + 1]; int bi[DK + 1];
#pragma unroll
    for (int q = 0; q <= DK; ++q) { bd[q] = __int_as_float(0x7f800000); bi[q] = INT_MAX; }
    for (int j = lo; j < hi; ++j) {
        const float dx = __fsub_rn(__ldg(&node_pos[3 * j]), vx), dy = __fsub_rn(__ldg(&node_pos[3 * j + 1]), vy), dz = __fsub_rn(__ldg(&node_pos[3 * j + 2]), vz);
        deform_insert(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))), j, bd, bi);
    }
    const double dmax = (double)bd[DK];
    double w[DK]; int id[DK]; double sum = 0.0;
#pragma unroll
    for (int q = 0; q < DK; ++q) {
        const int j = bi[q];
        const double ex = __dsub_rn(vx, (double)node_pos[3 * j]), ey = __dsub_rn(vy, (double)node_pos[3 * j + 1]), ez = __dsub_rn(vz, (double)node_pos[3 * j + 2]);
        const double dd = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez)));
        const double a = __dsub_rn(1.0, __ddiv_rn(dd, dmax));
        w[q] = __dmul_rn(a, a);
        id[q] = j;
        sum = __dadd_rn(sum, w[q]);
    }
    // the reference divides by 0 (NaN weights) when the k nearest all lie at dMax (quirk R3); equal weights keep the vertex on its
    // nodes.  A sum that is not > 0 (also NaN, from a non-finite point) takes the same branch.
#pragma unroll
    for (int q = 0; q < DK; ++q) w[q] = sum > 0.0 ? __ddiv_rn(w[q], sum) : 1.0 / DK;
    // VertexWeightMap::sort: by node id
#pragma unroll
    for (int a = 1; a < DK; ++a)
#pragma unroll
        for (int b = DK - 1; b >= a; --b)
            if (id[b - 1] > id[b]) { const int ti = id[b]; id[b] = id[b - 1]; id[b - 1] = ti; const double tw = w[b]; w[b] = w[b - 1]; w[b - 1] = tw; }
    ids[i] = make_int4(id[0], id[1], id[2], id[3]);
    double2* wo = (double2*)(weights + 4 * i);
    wo[0] = make_double2(w[0], w[1]); wo[1] = make_double2(w[2], w[3]);
}

// ---- fixed-order block reduction --------------------------------------------------------------------------------------------
template <int T>
__device__ double block_sum(double v, double* red)
{
    red[threadIdx.x] = v;
    __syncthreads();
#pragma unroll
    for (int s = T / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
}

// E_rot of one node (sparseResidual :942-958, sparseJacobian :786-829): 6 residuals, and the 6 x 9 Jacobian on the rotation
__device__ __forceinline__ void rot_residual(const double* x, double* r)
{
    const double* c0 = x; const double* c1 = x + 3; const double* c2 = x + 6;
    r[0] = c0[0] * c1[0] + c0[1] * c1[1] + c0[2] * c1[2];
    r[1] = c0[0] * c2[0] + c0[1] * c2[1] + c0[2] * c2[2];
    r[2] = c1[0] * c2[0] + c1[1] * c2[1] + c1[2] * c2[2];
    r[3] = c0[0] * c0[0] + c0[1] * c0[1] + c0[2] * c0[2] - 1.0;
    r[4] = c1[0] * c1[0] + c1[1] * c1[1] + c1[2] * c1[2] - 1.0;
    r[5] = c2[0] * c2[0] + c2[1] * c2[1] + c2[2] * c2[2] - 1.0;
}
__device__ __forceinline__ double rot_jac(const double* x, int row, int p)      // d r_row / d x[p], p < 9
{
    const int col = p / 3, e = p % 3;
    switch (row) {
    case 0: return col == 0 ? x[3 + e] : col == 1 ? x[e] : 0.0;
    case 1: return col == 0 ? x[6 + e] : col == 2 ? x[e] : 0.0;
    case 2: return col == 1 ? x[6 + e] : col == 2 ? x[3 + e] : 0.0;
    case 3: return col == 0 ? 2.0 * x[e] : 0.0;
    case 4: return col == 1 ? 2.0 * x[3 + e] : 0.0;
    default: return col == 2 ? 2.0 * x[6 + e] : 0.0;
    }
}

struct TermsDev {
    const int* node;         // [T][DK], -1 = unused slot
    const double* u;         // [T][DK][4]
    const double* c;         // [T][3]
    int n_terms, n_con_first;        // terms [n_con_first, n_terms) are constraints
    const int* list_off;     // [n + 1]: node a's terms are list_term[list_off[a] .. list_off[a+1]), ascending
    const int* list_term; const int* list_slot;
};

// Residual of every term at the current unknowns, |r|^2 and the constraint part of it.  One CTA.
__global__ void __launch_bounds__(RES_THREADS)
deform_residual_kernel(const double* __restrict__ x, int n, TermsDev t, double* __restrict__ r_rot, double* __restrict__ r_lin, double* __restrict__ out)
{
    __shared__ double red[RES_THREADS];
    double all = 0.0, con = 0.0;
    for (int a = threadIdx.x; a < n; a += RES_THREADS) {
        double r[6]; rot_residual(x + 12 * a, r);
        for (int q = 0; q < 6; ++q) { r_rot[6 * a + q] = r[q]; all += r[q] * r[q]; }
    }
    for (int k = threadIdx.x; k < t.n_terms; k += RES_THREADS) {
        double r[3] = {t.c[3 * k], t.c[3 * k + 1], t.c[3 * k + 2]};
        for (int sl = 0; sl < DK; ++sl) {
            const int j = t.node[DK * k + sl];
            if (j < 0) continue;
            const double* u = t.u + 4 * (DK * k + sl); const double* xj = x + 12 * j;
            for (int e = 0; e < 3; ++e) r[e] += u[0] * xj[e] + u[1] * xj[3 + e] + u[2] * xj[6 + e] + u[3] * xj[9 + e];
        }
        double sq = 0.0;
        for (int e = 0; e < 3; ++e) { r_lin[3 * k + e] = r[e]; sq += r[e] * r[e]; }
        all += sq;
        if (k >= t.n_con_first) con += sq;
    }
    all = block_sum<RES_THREADS>(all, red);
    con = block_sum<RES_THREADS>(con, red);
    if (threadIdx.x == 0) { out[2] = all; out[3] = con; }
}

// Block row a of J^T J (blocks (a, a-d), d = 0..19) and of -J^T r.  One CTA per node, thread (d, m, m').
__global__ void __launch_bounds__(ASM_THREADS)
deform_assemble_kernel(const double* __restrict__ x, int n, TermsDev t, const double* __restrict__ r_rot, const double* __restrict__ r_lin,
                       double* __restrict__ H, double* __restrict__ rhs)
{
    __shared__ double D[144];
    const int a = blockIdx.x;
    const int d = threadIdx.x / 16, m = (threadIdx.x / 4) % 4, m2 = threadIdx.x % 4;
    const int b = a - d;
    const int l0 = t.list_off[a], l1 = t.list_off[a + 1];
    if (threadIdx.x < 144) D[threadIdx.x] = 0.0;
    __syncthreads();
    if (b >= 0) {
        double acc = 0.0;
        for (int l = l0; l < l1; ++l) {
            const int k = t.list_term[l], sa = t.list_slot[l];
            for (int sl = 0; sl < DK; ++sl)
                if (t.node[DK * k + sl] == b) acc += t.u[4 * (DK * k + sa) + m] * t.u[4 * (DK * k + sl) + m2];
        }
        double* blk = H + ((size_t)a * BW + d) * 144;
        for (int e = 0; e < 3; ++e) {
            const int p = 3 * m + e, q = 3 * m2 + e;
            if (d == 0) D[p * 12 + q] = acc; else blk[p * 12 + q] = acc;
        }
    }
    __syncthreads();
    const double* xa = x + 12 * a;
    if (threadIdx.x < 81) {
        const int p = threadIdx.x / 9, q = threadIdx.x % 9;
        double acc = 0.0;
        for (int row = 0; row < 6; ++row) acc += rot_jac(xa, row, p) * rot_jac(xa, row, q);
        D[p * 12 + q] += acc;
    }
    __syncthreads();
    if (threadIdx.x < 144) H[(size_t)a * BW * 144 + threadIdx.x] = D[threadIdx.x];
    if (threadIdx.x >= 160 && threadIdx.x < 172) {
        const int p = threadIdx.x - 160, mm = p / 3, e = p % 3;
        double g = 0.0;
        for (int l = l0; l < l1; ++l) { const int k = t.list_term[l], sa = t.list_slot[l]; g += t.u[4 * (DK * k + sa) + mm] * r_lin[3 * k + e]; }
        if (p < 9) for (int row = 0; row < 6; ++row) g += rot_jac(xa, row, p) * r_rot[6 * a + row];
        rhs[12 * a + p] = -g;
    }
}

// Block-banded Cholesky H = L L^T in place (right-looking over block columns), L y = rhs, L^T delta = y, x += delta, |delta|^2.
// One CTA: the column panel lives in shared memory, the trailing window of the band in global memory (L2-resident).  A pivot that is
// not positive (or not finite) stops the sweep with out[1] = 1 and leaves x unchanged.
__global__ void __launch_bounds__(SOLVE_THREADS, 1)
deform_solve_kernel(double* __restrict__ H, double* __restrict__ rhs, int n, double* __restrict__ x, double* __restrict__ out)
{
    const int B = BW - 1;
    __shared__ double D[144];
    __shared__ double P[DEFORM_BAND][144];
    __shared__ double part[DEFORM_BAND][12];
    __shared__ double red[SOLVE_THREADS];
    __shared__ unsigned char pair_i[DEFORM_BAND * BW / 2], pair_l[DEFORM_BAND * BW / 2];
    __shared__ int fail;
    const int tid = threadIdx.x;
    if (tid == 0) {
        fail = 0;
        int q = 0;
        for (int i = 0; i < B; ++i) for (int l = 0; l <= i; ++l) { pair_i[q] = (unsigned char)i; pair_l[q] = (unsigned char)l; ++q; }
    }
    __syncthreads();
    for (int j = 0; j < n; ++j) {
        const int nb = min(B, n - 1 - j);
        double* Hj = H + (size_t)j * BW * 144;
        if (tid < 144) D[tid] = Hj[tid];
        __syncthreads();
        if (tid < 32) {                                      // 12 x 12 Cholesky of the diagonal block, one warp, lane = row
            const int r = tid;
            for (int c = 0; c < 12; ++c) {
                const double piv = D[c * 12 + c];
                __syncwarp();
                if (!(piv > 0.0) || !isfinite(piv)) { if (r == 0) fail = 1; break; }
                const double lc = sqrt(piv);
                if (r == c) D[c * 12 + c] = lc;
                if (r > c && r < 12) D[r * 12 + c] = D[r * 12 + c] / lc;
                __syncwarp();
                if (r > c && r < 12) for (int s = c + 1; s <= r; ++s) D[r * 12 + s] -= D[r * 12 + c] * D[s * 12 + c];
                __syncwarp();
            }
        }
        __syncthreads();
        if (fail) break;
        if (tid < 144) Hj[tid] = D[tid];
        if (tid < nb * 12) {                                 // panel: L(i, j) = H(i, j) L_jj^-T, one row per thread
            const int bi = tid / 12, r = tid % 12, i = j + 1 + bi;
            double* row = H + ((size_t)i * BW + (i - j)) * 144 + r * 12;
            double xr[12];
#pragma unroll
            for (int c = 0; c < 12; ++c) {
                double v = row[c];
#pragma unroll
                for (int s = 0; s < c; ++s) v -= xr[s] * D[c * 12 + s];
                xr[c] = v / D[c * 12 + c];
            }
#pragma unroll
            for (int c = 0; c < 12; ++c) { row[c] = xr[c]; P[bi][r * 12 + c] = xr[c]; }
        }
        __syncthreads();
        const int np = nb * (nb + 1) / 2;                    // trailing update H(i, l) -= L(i, j) L(l, j)^T, j < l <= i <= j + nb
        for (int idx = tid; idx < np * 144; idx += SOLVE_THREADS) {
            const int pr = idx / 144, e = idx % 144, p = e / 12, q = e % 12;
            const int bi = pair_i[pr], bl = pair_l[pr];
            const int i = j + 1 + bi, l = j + 1 + bl;
            double acc = 0.0;
#pragma unroll
            for (int c = 0; c < 12; ++c) acc += P[bi][p * 12 + c] * P[bl][q * 12 + c];
            H[((size_t)i * BW + (i - l)) * 144 + e] -= acc;
        }
        __syncthreads();
    }
    if (fail) {
        if (tid == 0) { out[0] = 0.0; out[1] = 1.0; }
        return;
    }
    // forward: L y = rhs (in place)
    for (int j = 0; j < n; ++j) {
        const int nb = min(B, n - 1 - j);
        const double* L = H + (size_t)j * BW * 144;
        if (tid == 0) {
            for (int r = 0; r < 12; ++r) {
                double v = rhs[12 * j + r];
                for (int s = 0; s < r; ++s) v -= L[r * 12 + s] * rhs[12 * j + s];
                rhs[12 * j + r] = v / L[r * 12 + r];
            }
        }
        __syncthreads();
        if (tid < nb * 12) {
            const int bi = tid / 12, r = tid % 12, i = j + 1 + bi;
            const double* row = H + ((size_t)i * BW + (i - j)) * 144 + r * 12;
            double acc = 0.0;
#pragma unroll
            for (int c = 0; c < 12; ++c) acc += row[c] * rhs[12 * j + c];
            rhs[12 * i + r] -= acc;
        }
        __syncthreads();
    }
    // backward: L^T delta = y (in place)
    for (int j = n - 1; j >= 0; --j) {
        const int nb = min(B, n - 1 - j);
        if (tid < nb * 12) {
            const int bi = tid / 12, r = tid % 12, i = j + 1 + bi;
            const double* blk = H + ((size_t)i * BW + (i - j)) * 144;
            double acc = 0.0;
#pragma unroll
            for (int q = 0; q < 12; ++q) acc += blk[q * 12 + r] * rhs[12 * i + q];
            part[bi][r] = acc;
        }
        __syncthreads();
        if (tid == 0) {
            const double* L = H + (size_t)j * BW * 144;
            for (int r = 11; r >= 0; --r) {
                double v = rhs[12 * j + r];
                for (int bi = 0; bi < nb; ++bi) v -= part[bi][r];
                for (int s = r + 1; s < 12; ++s) v -= L[s * 12 + r] * rhs[12 * j + s];
                rhs[12 * j + r] = v / L[r * 12 + r];
            }
        }
        __syncthreads();
    }
    double sq = 0.0;
    for (int k = tid; k < 12 * n; k += SOLVE_THREADS) { const double dl = rhs[k]; x[k] += dl; sq += dl * dl; }
    sq = block_sum<SOLVE_THREADS>(sq, red);
    if (tid == 0) { out[0] = sq; out[1] = 0.0; }
}

// Per node: R row-major, R^-T (Eigen's rotation.inverse().transpose(): cofactors over the determinant), g, g + t
struct NodeTable { double R[9]; double Rit[9]; double g[3]; double gt[3]; };

__global__ void deform_node_table_kernel(const float* __restrict__ node_pos, const double* __restrict__ x, int n, NodeTable* __restrict__ tab)
{
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n) return;
    const double* xa = x + 12 * a;
    NodeTable t;
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) t.R[3 * r + c] = xa[3 * c + r];
    const double* m = t.R;
    double cof[9];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
            cof[3 * r + c] = m[3 * ((r + 1) % 3) + (c + 1) % 3] * m[3 * ((r + 2) % 3) + (c + 2) % 3]
                           - m[3 * ((r + 1) % 3) + (c + 2) % 3] * m[3 * ((r + 2) % 3) + (c + 1) % 3];
    const double det = m[0] * cof[0] + m[1] * cof[1] + m[2] * cof[2];
    for (int k = 0; k < 9; ++k) t.Rit[k] = cof[k] / det;               // (adj / det)^T = cof / det
    for (int e = 0; e < 3; ++e) { t.g[e] = (double)node_pos[3 * a + e]; t.gt[e] = t.g[e] + xa[9 + e]; }
    tab[a] = t;
}

// computeVertexPosition (:1028-1054): position sum_j w_j (R_j (v - g_j) + g_j + t_j), normal sum_j w_j R_j^-T n normalised (a zero
// normal stays zero), FP64, written as float; every other byte of the record is copied.  Normal at float offset NO.
template <int WORDS, int NO>
__global__ void __launch_bounds__(256)
deform_apply_kernel(const float4* __restrict__ in, float4* __restrict__ out, const int4* __restrict__ ids, const double* __restrict__ weights,
                    const NodeTable* __restrict__ tab, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float4 w4[WORDS];
#pragma unroll
    for (int q = 0; q < WORDS; ++q) w4[q] = __ldcs(&in[i * WORDS + q]);
    float* f = (float*)w4;
    const double v[3] = {f[0], f[1], f[2]}, nv[3] = {f[NO], f[NO + 1], f[NO + 2]};
    const int4 id4 = __ldcs(&ids[i]);
    const double2 wa = __ldcs((const double2*)(weights + 4 * i)), wb = __ldcs((const double2*)(weights + 4 * i) + 1);
    const int id[4] = {id4.x, id4.y, id4.z, id4.w};
    const double w[4] = {wa.x, wa.y, wb.x, wb.y};
    double p[3] = {0, 0, 0}, nn[3] = {0, 0, 0};
#pragma unroll
    for (int q = 0; q < DK; ++q) {
        const NodeTable* t = tab + id[q];
        const double d[3] = {v[0] - t->g[0], v[1] - t->g[1], v[2] - t->g[2]};
#pragma unroll
        for (int e = 0; e < 3; ++e) {
            p[e] += w[q] * (t->R[3 * e] * d[0] + t->R[3 * e + 1] * d[1] + t->R[3 * e + 2] * d[2] + t->gt[e]);
            nn[e] += w[q] * (t->Rit[3 * e] * nv[0] + t->Rit[3 * e + 1] * nv[1] + t->Rit[3 * e + 2] * nv[2]);
        }
    }
    const double l2 = nn[0] * nn[0] + nn[1] * nn[1] + nn[2] * nn[2];
    const double inv = l2 > 0.0 ? 1.0 / sqrt(l2) : 0.0;
    for (int e = 0; e < 3; ++e) { f[e] = (float)p[e]; f[NO + e] = (float)(nn[e] * inv); }
#pragma unroll
    for (int q = 0; q < WORDS; ++q) __stcs(&out[i * WORDS + q], w4[q]);
}

size_t point_stride(int kind) { return kind == 0 ? sizeof(kt_point_xyzrgbnormal) : kind == 1 ? sizeof(kt_mesh_vertex) : 12; }

} // namespace

int deform_weights(const float* node_pos, const uint64_t* node_times, int n_nodes, const void* pts, int kind, const uint64_t* times, size_t n,
                   int32_t* ids, double* weights, cudaStream_t s)
{
    if (n_nodes < DK + 1) { set_error("deform_weights: %d nodes, need at least %d", n_nodes, DK + 1); return KT_ERR_STATE; }
    if (kind < 0 || kind > 2) { set_error("deform_weights: kind %d", kind); return KT_ERR_INVALID; }
    if (!n) return 0;
    const size_t nb = (n + 255) / 256;
    deform_weight_kernel<<<(unsigned int)nb, 256, 0, s>>>(node_pos, node_times, n_nodes, (const unsigned char*)pts, point_stride(kind), times, n,
                                                          (int4*)ids, weights);
    KT_LAUNCH_CHECK();
    return 0;
}

int deform_optimise(const float* node_pos, int n, const float* src, const double* dst, const int32_t* cids, const double* cw, size_t m,
                    double* x_dev, kt_deform_report* res, cudaStream_t s)
{
    std::memset(res, 0, sizeof(*res));
    res->nodes = n; res->constraints = (int)m;
    if (n < DK + 1) { set_error("deform_optimise: %d nodes, need at least %d", n, DK + 1); return KT_ERR_STATE; }
    if (m == 0) { set_error("deform_optimise: no constraints"); return KT_ERR_INVALID; }
    if (deform_first_non_finite(node_pos, 3 * (size_t)n) >= 0 || deform_first_non_finite(src, 3 * m) >= 0 ||
        deform_first_non_finite(dst, 3 * m) >= 0 || deform_first_non_finite(cw, (size_t)DK * m) >= 0) {
        set_error("deform_optimise: a node position, constraint source, target or weight is not finite"); return KT_ERR_INVALID;
    }
    // ---- the affine terms (see the file header), node-major lists, band check ----
    std::vector<int> noff, nbr; deform_connect_seq(n, DK, noff, nbr);
    const size_t n_reg = nbr.size(), T = n_reg + m;
    std::vector<int> tnode(T * DK, -1); std::vector<double> tu(T * DK * 4, 0.0), tc(T * 3, 0.0);
    auto g = [&](int j, int e) { return (double)node_pos[3 * j + e]; };
    const double sreg = std::sqrt(10.0), scon = std::sqrt(100.0);        // wReg, wCon (DeformationGraph.cpp:24-26)
    int band = 0;
    size_t k = 0;
    for (int j = 0; j < n; ++j)
        for (int q = noff[j]; q < noff[j + 1]; ++q, ++k) {                 // sparseResidual :963-973, sparseJacobian :833-881
            const int nn = nbr[q];
            tnode[DK * k] = j; tnode[DK * k + 1] = nn;
            for (int e = 0; e < 3; ++e) { tu[4 * DK * k + e] = sreg * (g(nn, e) - g(j, e)); tc[3 * k + e] = sreg * (g(j, e) - g(nn, e)); }
            tu[4 * DK * k + 3] = sreg; tu[4 * (DK * k + 1) + 3] = -sreg;
            band = std::max(band, std::abs(nn - j));
        }
    for (size_t l = 0; l < m; ++l, ++k) {                                  // sparseResidual :975-985, sparseJacobian :883-923
        double sw[3] = {0, 0, 0};
        int lo = n, hi = -1;
        for (int q = 0; q < DK; ++q) {
            const int j = cids[DK * l + q]; const double w = cw[DK * l + q];
            if (j < 0 || j >= n || (q && j <= cids[DK * l + q - 1])) { set_error("deform_optimise: constraint %zu has bad node ids", l); return KT_ERR_INVALID; }
            tnode[DK * k + q] = j;
            for (int e = 0; e < 3; ++e) { tu[4 * (DK * k + q) + e] = scon * w * ((double)src[3 * l + e] - g(j, e)); sw[e] += w * g(j, e); }
            tu[4 * (DK * k + q) + 3] = scon * w;
            lo = std::min(lo, j); hi = std::max(hi, j);
        }
        for (int e = 0; e < 3; ++e) tc[3 * k + e] = scon * (sw[e] - dst[3 * l + e]);
        band = std::max(band, hi - lo);
    }
    res->band = band;
    if (band > DEFORM_BAND) { set_error("deform_optimise: a term spans %d node blocks, the band holds %d", band, DEFORM_BAND); return KT_ERR_INVALID; }
    std::vector<int> loff(n + 1, 0), lterm, lslot;
    for (size_t t = 0; t < T; ++t) for (int q = 0; q < DK; ++q) if (tnode[DK * t + q] >= 0) ++loff[tnode[DK * t + q] + 1];
    for (int j = 0; j < n; ++j) loff[j + 1] += loff[j];
    lterm.resize(loff[n]); lslot.resize(loff[n]);
    { std::vector<int> fill(loff.begin(), loff.end() - 1);
      for (size_t t = 0; t < T; ++t) for (int q = 0; q < DK; ++q) { const int j = tnode[DK * t + q]; if (j >= 0) { lterm[fill[j]] = (int)t; lslot[fill[j]] = q; ++fill[j]; } } }
    std::vector<double> x0((size_t)n * 12, 0.0);
    for (int j = 0; j < n; ++j) { x0[12 * j] = 1.0; x0[12 * j + 4] = 1.0; x0[12 * j + 8] = 1.0; }

    // ---- device buffers (once per call: the deformation runs once per loop closure) ----
    Allocations mem(s); const char* W = "deform_optimise scratch";
    int *d_node, *d_off, *d_term, *d_slot; double *d_u, *d_c, *d_rrot, *d_rlin, *d_H, *d_rhs, *d_out;
    const size_t hbytes = (size_t)n * BW * 144 * sizeof(double);
    if (mem.device(&d_node, T * DK, W) || mem.device(&d_off, n + 1, W) || mem.device(&d_term, lterm.size(), W) || mem.device(&d_slot, lslot.size(), W) ||
        mem.device(&d_u, tu.size(), W) || mem.device(&d_c, tc.size(), W) || mem.device(&d_rrot, (size_t)n * 6, W) || mem.device(&d_rlin, T * 3, W) ||
        mem.device(&d_H, (size_t)n * BW * 144, W) || mem.device(&d_rhs, (size_t)n * 12, W) || mem.device(&d_out, 4, W)) return KT_ERR_CUDA;
    KT_CUDA(cudaMemcpyAsync(d_node, tnode.data(), tnode.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(d_off, loff.data(), loff.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(d_term, lterm.data(), lterm.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(d_slot, lslot.data(), lslot.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(d_u, tu.data(), tu.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(d_c, tc.data(), tc.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(x_dev, x0.data(), x0.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    TermsDev td; td.node = d_node; td.u = d_u; td.c = d_c; td.n_terms = (int)T; td.n_con_first = (int)n_reg;
    td.list_off = d_off; td.list_term = d_term; td.list_slot = d_slot;
    double out[4];
    auto residual = [&]() -> int {
        deform_residual_kernel<<<1, RES_THREADS, 0, s>>>(x_dev, n, td, d_rrot, d_rlin, d_out);
        KT_LAUNCH_CHECK();
        return 0;
    };
    auto readback = [&]() -> int {
        KT_CUDA(cudaMemcpyAsync(out, d_out, sizeof(out), cudaMemcpyDeviceToHost, s));
        KT_CUDA(cudaStreamSynchronize(s));
        return 0;
    };
    // optimiseGraphSparse (:714-774)
    int rr = residual(); if (rr) return rr;
    rr = readback(); if (rr) return rr;
    const float graph_error = (float)(std::sqrt(out[3]) / (double)m);
    res->constraint_error = graph_error;
    res->initial_error = res->final_error = out[2];
    // left undeformed: the identity
    auto identity = [&]() -> int { KT_CUDA(cudaMemcpy(x_dev, x0.data(), x0.size() * sizeof(double), cudaMemcpyHostToDevice)); return 0; };
    if (graph_error < 0.1) return identity();                          // "Not deforming, constraint error insignificant"
    double error = out[2], last = error;
    int iter = 0;
    while (iter < 10) {
        ++iter;
        KT_CUDA(cudaMemsetAsync(d_H, 0, hbytes, s));
        deform_assemble_kernel<<<n, ASM_THREADS, 0, s>>>(x_dev, n, td, d_rrot, d_rlin, d_H, d_rhs);
        KT_LAUNCH_CHECK();
        deform_solve_kernel<<<1, SOLVE_THREADS, 0, s>>>(d_H, d_rhs, n, x_dev, d_out);
        KT_LAUNCH_CHECK();
        rr = residual(); if (rr) return rr;
        rr = readback(); if (rr) return rr;
        res->iterations = iter;
        if (out[1] != 0.0) { res->solver_failed = 1; return identity(); }
        error = out[2];
        res->final_error = error;
        const double diff = error - last;
        if (std::sqrt(out[0]) < 1e-2 || error < 1e-3 || std::fabs(diff) < 1e-5 * error) break;
        last = error;
    }
    res->deformed = 1;
    return 0;
}

int deform_apply(const float* node_pos, const double* x, int n_nodes, const int32_t* ids, const double* weights, const void* in, void* out,
                 int kind, size_t n, cudaStream_t s)
{
    if (kind != 0 && kind != 1) { set_error("deform_apply: kind %d", kind); return KT_ERR_INVALID; }
    if (!n) return 0;
    NodeTable* tab = 0;
    const size_t bytes = (size_t)n_nodes * sizeof(NodeTable);
    const cudaError_t e = cudaMallocAsync((void**)&tab, bytes, s);
    if (e != cudaSuccess) return refused(e, "cudaMallocAsync", "deform_apply node table", bytes);
    deform_node_table_kernel<<<(n_nodes + 127) / 128, 128, 0, s>>>(node_pos, x, n_nodes, tab);
    int r = kt::cuda_check(cudaGetLastError(), "kernel launch", __FILE__, __LINE__); ++g_launches;
    if (!r) {
        const unsigned int nb = (unsigned int)((n + 255) / 256);
        if (kind == 0) deform_apply_kernel<3, 4><<<nb, 256, 0, s>>>((const float4*)in, (float4*)out, (const int4*)ids, weights, tab, n);
        else deform_apply_kernel<2, 3><<<nb, 256, 0, s>>>((const float4*)in, (float4*)out, (const int4*)ids, weights, tab, n);
        r = kt::cuda_check(cudaGetLastError(), "kernel launch", __FILE__, __LINE__); ++g_launches;
    }
    cudaFreeAsync(tab, s);
    return r;
}

} // namespace kt
