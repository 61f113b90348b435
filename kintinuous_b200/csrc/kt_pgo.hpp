// kintinuous_b200 -- the host side of loop closure: the dense pose graph as an iSAM-style pose graph, CUDA-free (CPU-tested through
// tests/cpp/pgo_host.cpp against oracle/pgo_oracle.py).  The Gauss-Newton solve is in kt_pgo.cu.
//
// Replaces (reference, src/backend/):
//   Deformation::addCameraCamera             Deformation.cpp:130-171  node selection (-fl / -dg, isLoopPose, the finalised last pose)
//   iSAMInterface::addCameraCameraConstraint iSAMInterface.cpp:44-83  odometry measurement: prev^-1 curr in float, M conjugation, float
//                                                                      quaternion, then FP64
//   iSAMInterface::addLoopConstraint         iSAMInterface.cpp:85-105 loop measurement M C M^-1 in FP64
//   iSAMInterface::cameraNode                iSAMInterface.cpp:107-134 the prior on the first node (anchored at the tracked pose here,
//                                                                      see DESIGN quirk R4)
// Pose3d (iSAM's slam3d.h, restated, unpinned): vector() = (x, y, z, yaw, pitch, roll) with R = Rz(yaw) Ry(pitch) Rx(roll).
#pragma once
#include "kt_deform.hpp"
#include "kt_posegraph.hpp"
#include <cmath>
#include <cstdint>
#include <cstddef>
#include <vector>
#include <algorithm>

namespace kt {

static const int PGO_MAX_LOOPS = 64;
static const int PGO_MAX_NODES = 1 << 18;
static const int PGO_SEG = 64;              // fixed segment boundaries of the elimination, every PGO_SEG nodes of a level

// One factor.  i = -1: the prior on node j, z = the anchor pose's vector(); else (p_j - p_i).vector() - z.  Layout = kt_pgo_factor.
struct PgoFactor { int32_t i, j; double z[6]; };

// transformation2isam (iSAMInterface.cpp:23-29): isam = M cam M^-1
static const double PGO_M[9] = {0, 0, 1, -1, 0, 0, 0, -1, 0};

// (-pi, pi]
inline double pgo_wrap(double a)
{
    double r = std::fmod(a + M_PI, 2.0 * M_PI);
    if (r <= 0.0) r += 2.0 * M_PI;
    return r - M_PI;
}

// yaw, pitch, roll of a row-major rotation (R = Rz Ry Rx)
inline void pgo_ypr(const double* R, double* ypr)
{
    ypr[0] = std::atan2(R[3], R[0]);
    ypr[1] = std::atan2(-R[6], std::sqrt(R[7] * R[7] + R[8] * R[8]));
    ypr[2] = std::atan2(R[7], R[8]);
}

inline void pgo_rot(const double* ypr, double* R)
{
    const double cy = std::cos(ypr[0]), sy = std::sin(ypr[0]), cp = std::cos(ypr[1]), sp = std::sin(ypr[1]);
    const double cr = std::cos(ypr[2]), sr = std::sin(ypr[2]);
    R[0] = cy * cp; R[1] = cy * sp * sr - sy * cr; R[2] = cy * sp * cr + sy * sr;
    R[3] = sy * cp; R[4] = sy * sp * sr + cy * cr; R[5] = sy * sp * cr - cy * sr;
    R[6] = -sp;     R[7] = cp * sr;                R[8] = cp * cr;
}

// M A M^T for a row-major 3 x 3 A (M is a signed permutation, so this is exact), and M v
inline void pgo_to_isam_R(const double* A, double* out)
{
    double t[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double s = 0; for (int k = 0; k < 3; ++k) s += PGO_M[3 * r + k] * A[3 * k + c]; t[3 * r + c] = s; }
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double s = 0; for (int k = 0; k < 3; ++k) s += t[3 * r + k] * PGO_M[3 * c + k]; out[3 * r + c] = s; }
}
inline void pgo_from_isam_R(const double* A, double* out)
{
    double t[9];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double s = 0; for (int k = 0; k < 3; ++k) s += PGO_M[3 * k + r] * A[3 * k + c]; t[3 * r + c] = s; }
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { double s = 0; for (int k = 0; k < 3; ++k) s += t[3 * r + k] * PGO_M[3 * k + c]; out[3 * r + c] = s; }
}
inline void pgo_to_isam_t(const double* v, double* out) { for (int r = 0; r < 3; ++r) out[r] = PGO_M[3 * r] * v[0] + PGO_M[3 * r + 1] * v[1] + PGO_M[3 * r + 2] * v[2]; }
inline void pgo_from_isam_t(const double* v, double* out) { for (int r = 0; r < 3; ++r) out[r] = PGO_M[r] * v[0] + PGO_M[3 + r] * v[1] + PGO_M[6 + r] * v[2]; }

// Node poses are 4 x 4 row-major FP64 (R in [0..2], [4..6], [8..10], t in [3], [7], [11]).
inline void pgo_split(const double* X, double* R, double* t) { for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) R[3 * r + c] = X[4 * r + c]; t[r] = X[4 * r + 3]; } }
inline void pgo_join(const double* R, const double* t, double* X)
{
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) X[4 * r + c] = R[3 * r + c]; X[4 * r + 3] = t[r]; }
    X[12] = X[13] = X[14] = 0.0; X[15] = 1.0;
}
// A tracked float pose (world frame) as an FP64 node pose in the isam frame, M P M^-1, and back
inline void pgo_pose_to_isam(const float* P, double* X)
{
    double R[9], t[3], Ri[9], ti[3];
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) R[3 * r + c] = P[4 * r + c]; t[r] = P[4 * r + 3]; }
    pgo_to_isam_R(R, Ri); pgo_to_isam_t(t, ti); pgo_join(Ri, ti, X);
}
inline void pgo_pose_from_isam(const double* X, double* P)
{
    double R[9], t[3], Rw[9], tw[3];
    pgo_split(X, R, t); pgo_from_isam_R(R, Rw); pgo_from_isam_t(t, tw); pgo_join(Rw, tw, P);
}
inline void pgo_vector(const double* X, double* v6) { double R[9]; pgo_split(X, R, v6); pgo_ypr(R, v6 + 3); }

// addCameraCameraConstraint (:60-76): delta = prev^-1 curr in float (the rigid inverse [R^T | -R^T t]; Eigen's general 4 x 4 inverse
// may differ in the last bit), d = M delta M^-1 (exact), Eigen::Quaternionf(d's rotation), then isam::Pose3d(trans, Quaterniond(q)) in
// FP64: the rotation of the unnormalised quaternion (Eigen's toRotationMatrix) and its yaw / pitch / roll.
inline void pgo_odometry_z(const float* prev, const float* curr, double* z)
{
    float inv[16] = {0};
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) inv[4 * r + c] = prev[4 * c + r];
        const float s = (prev[r] * prev[3] + prev[4 + r] * prev[7]) + prev[8 + r] * prev[11];
        inv[4 * r + 3] = -s;
    }
    inv[15] = 1.0f;
    float d[16];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) d[4 * r + c] = ((inv[4 * r] * curr[c] + inv[4 * r + 1] * curr[4 + c]) + inv[4 * r + 2] * curr[8 + c]) + inv[4 * r + 3] * curr[12 + c];
    float Ri[9], ti[3];
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) {
            float s = 0.0f;                      // M d M^T: every product has one nonzero term, exact in float
            for (int k = 0; k < 3; ++k) for (int l = 0; l < 3; ++l) if (PGO_M[3 * r + k] != 0.0 && PGO_M[3 * c + l] != 0.0) s = (float)(PGO_M[3 * r + k] * PGO_M[3 * c + l]) * d[4 * k + l];
            Ri[3 * r + c] = s;
        }
        float s = 0.0f;
        for (int k = 0; k < 3; ++k) if (PGO_M[3 * r + k] != 0.0) s = (float)PGO_M[3 * r + k] * d[4 * k + 3];
        ti[r] = s;
    }
    float q[4];
    quaternion_from_rotation(Ri, q);
    const double x = q[0], y = q[1], zq = q[2], w = q[3];
    // Eigen QuaternionBase::toRotationMatrix
    const double tx = 2 * x, ty = 2 * y, tz = 2 * zq, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * zq;
    const double R[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
    for (int e = 0; e < 3; ++e) z[e] = (double)ti[e];
    pgo_ypr(R, z + 3);
}

// addLoopConstraint (:95): Pose3d(M C M^-1) in FP64; C row-major 4 x 4
inline void pgo_loop_z(const double* C, double* z)
{
    double R[9], t[3], Ri[9];
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) R[3 * r + c] = C[4 * r + c]; t[r] = C[4 * r + 3]; }
    pgo_to_isam_R(R, Ri); pgo_to_isam_t(t, z);
    pgo_ypr(Ri, z + 3);
}

// Caller input of a loop constraint: finite, rotation within 1e-3 of orthonormal (max |R^T R - I|).  0 when acceptable.
inline int pgo_check_constraint(const double* C)
{
    for (int k = 0; k < 16; ++k) if (!std::isfinite(C[k])) return 1;
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            const double s = C[a] * C[b] + C[4 + a] * C[4 + b] + C[8 + a] * C[8 + b];
            if (std::fabs(s - (a == b ? 1.0 : 0.0)) > 1e-3) return 2;
        }
    return 0;
}

// addCameraCamera (:134-170): with pose_spacing == 0 every dense pose; else the first, then each pose more than pose_spacing (float) from
// the last one taken, or flagged (a loop pose); the last dense pose always.  Returns the indices taken, ascending.
inline std::vector<int> pgo_select_nodes(const float* pos, const unsigned char* flagged, size_t n, float pose_spacing)
{
    std::vector<int> take;
    if (!n) return take;
    take.push_back(0);
    for (size_t i = 1; i < n; ++i)
        if (pose_spacing == 0.0f || flagged[i] || deform_dist_f(&pos[3 * take.back()], &pos[3 * i]) > pose_spacing) take.push_back((int)i);
    if (take.back() != (int)n - 1) take.push_back((int)n - 1);
    return take;
}

// The elimination plan.  Level 0 is the chain of nodes; the separators of a level are its first and last node, every PGO_SEG-th node
// and every loop endpoint; the nodes between two consecutive separators (a segment's interior) are eliminated, and the separators
// are the next level's chain.  The last level has no interior: it is solved densely together with the loop couplings.
struct PgoPlan {
    std::vector<int> n;                       // nodes per level
    std::vector<std::vector<int> > sep;       // sep[l][p]: node of level l that is node p of level l + 1 (levels 0 .. top - 1)
    std::vector<int> loop_i, loop_j;          // loop endpoints as nodes of the top level
    int top() const { return (int)n.size() - 1; }
};
inline PgoPlan pgo_plan(int n_nodes, const std::vector<int>& li, const std::vector<int>& lj)
{
    PgoPlan p;
    std::vector<int> keep(li); keep.insert(keep.end(), lj.begin(), lj.end());
    std::vector<int> at_i(li), at_j(lj);
    int n = n_nodes;
    p.n.push_back(n);
    for (;;) {
        std::vector<char> is(n, 0);
        is[0] = 1; is[n - 1] = 1;
        for (int k = 0; k < n; k += PGO_SEG) is[k] = 1;
        for (int k : keep) is[k] = 1;
        std::vector<int> sep, remap(n, -1);
        for (int k = 0; k < n; ++k) if (is[k]) { remap[k] = (int)sep.size(); sep.push_back(k); }
        if ((int)sep.size() == n) break;
        for (auto& k : keep) k = remap[k];
        for (auto& k : at_i) k = remap[k];
        for (auto& k : at_j) k = remap[k];
        p.sep.push_back(sep);
        n = (int)sep.size();
        p.n.push_back(n);
    }
    p.loop_i = at_i; p.loop_j = at_j;
    return p;
}

// The factor list of a chain: the prior on node 0 (anchor = node 0's pose), odometry k-1 -> k, then the loops.  Factor list checks
// of kt_op_pgo_optimise: 0 when the list has that shape, with every index in range and i != j.
inline int pgo_check_factors(const PgoFactor* f, int n_factors, int n_nodes)
{
    if (n_nodes < 2 || n_factors < n_nodes) return 1;
    if (f[0].i != -1 || f[0].j != 0) return 2;
    for (int k = 1; k < n_nodes; ++k) if (f[k].i != k - 1 || f[k].j != k) return 3;
    for (int l = n_nodes; l < n_factors; ++l) if (f[l].i < 0 || f[l].j < 0 || f[l].i >= n_nodes || f[l].j >= n_nodes || f[l].i == f[l].j) return 4;
    for (int l = 0; l < n_factors; ++l) for (int e = 0; e < 6; ++e) if (!std::isfinite(f[l].z[e])) return 5;
    return 0;
}

// Loop factors per node (CSR, ascending factor index): what pgo_assemble_kernel gathers besides the chain and the prior
inline void pgo_loop_csr(const PgoFactor* f, int n_factors, int n_nodes, std::vector<int>& off, std::vector<int>& idx)
{
    off.assign(n_nodes + 1, 0); idx.clear();
    for (int l = n_nodes; l < n_factors; ++l) { ++off[f[l].i + 1]; ++off[f[l].j + 1]; }
    for (int k = 0; k < n_nodes; ++k) off[k + 1] += off[k];
    idx.resize(off[n_nodes]);
    std::vector<int> fill(off.begin(), off.end() - 1);
    for (int l = n_nodes; l < n_factors; ++l) { idx[fill[f[l].i]++] = l; idx[fill[f[l].j]++] = l; }
}

} // namespace kt
