// kintinuous_b200 -- the host side of the embedded deformation graph, CUDA-free (CPU-tested through tests/cpp/deform_host.cpp against
// oracle/deform_oracle.py).  The kernels (weights, normal equations, banded Cholesky, apply) are in kt_deform.cu.
//
// Replaces (reference, src/backend/):
//   DeformationGraph::initialiseGraphPoses   DeformationGraph.cpp:51-86   node sampling from the dense pose graph
//   DeformationGraph::connectGraphSeq        DeformationGraph.cpp:217-271 sequential connectivity
//   DeformationGraph::weightVerticesSeq      DeformationGraph.cpp:454-498 the time -> nearest node lookup (with the clamp of quirk R2)
//   Deformation::addCameraLoop               Deformation.cpp:233-276     one position constraint per corrected camera pose
#pragma once
#include <cmath>
#include <cstdint>
#include <cstddef>
#include <vector>
#include <unordered_map>

namespace kt {

static const int DEFORM_K = 4;              // Deformation.cpp:469 (k of the graph and of every vertex's node set)
static const int DEFORM_LOOKBACK = 20;      // DeformationGraph.cpp:445: candidates per vertex
static const int DEFORM_BAND = 19;          // max(DEFORM_LOOKBACK - 1, DEFORM_K): block half-bandwidth of the normal equations

// ||a - b|| in float, as Eigen's (Vector3f - Vector3f).norm(): ((dx*dx + dy*dy) + dz*dz), correctly rounded sqrt
inline float deform_dist_f(const float* a, const float* b)
{
    const float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    volatile float s = dx * dx;              // volatile: no FMA contraction, the same bits as the device's __fmul_rn / __fadd_rn
    s = s + dy * dy;
    s = s + dz * dz;
    return std::sqrt((float)s);
}

// initialiseGraphPoses (:62-73): the first position, then every position more than pose_dist from the last one taken.
// pos: n x 3 float.  Returns the indices taken, ascending.
inline std::vector<int> deform_sample_nodes(const float* pos, size_t n, float pose_dist)
{
    std::vector<int> take;
    if (!n) return take;
    take.push_back(0);
    for (size_t i = 1; i < n; ++i)
        if (deform_dist_f(&pos[3 * take.back()], &pos[3 * i]) > pose_dist) take.push_back((int)i);
    return take;
}

// connectGraphSeq (:237-270): the first k/2 nodes connect to the first k+1 (themselves excepted), the middle ones to i-1, i+1, i-2, i+2,
// ..., the last k/2 to the last k+1.  Needs n >= k+1.  Flattened: neighbours of node i are out[off[i] .. off[i+1]).
inline void deform_connect_seq(int n, int k, std::vector<int>& off, std::vector<int>& out)
{
    off.assign(1, 0); out.clear();
    for (int i = 0; i < n; ++i) {
        if (i < k / 2) {
            for (int m = 0; m < k + 1; ++m) if (m != i) out.push_back(m);
        } else if (i < n - k / 2) {
            for (int m = 0; m < k / 2; ++m) { out.push_back(i - (m + 1)); out.push_back(i + (m + 1)); }
        } else {
            for (int m = n - (k + 1); m < n; ++m) if (m != i) out.push_back(m);
        }
        off.push_back((int)out.size());
    }
}

// weightVerticesSeq's binary search and nearest-in-time choice (:454-498).  The reference reads times[imin] with imin == n and
// times[imax] with imax == -1 when t lies outside [times[0], times[n-1]] (quirk R2); both indices are clamped to [0, n) here.
#if defined(__CUDACC__)
__host__ __device__
#endif
inline int deform_nearest_node(const uint64_t* times, int n, uint64_t t)
{
    int imin = 0, imax = n - 1, imid = (imin + imax) / 2;
    while (imax >= imin) {
        imid = (imin + imax) / 2;
        if (times[imid] < t) imin = imid + 1;
        else if (times[imid] > t) imax = imid - 1;
        else break;
    }
    if (imin > n - 1) imin = n - 1;
    if (imax < 0) imax = 0;
    const uint64_t ta = times[imin], tm = times[imid], tb = times[imax];
    const uint64_t da = ta > t ? ta - t : t - ta, dm = tm > t ? tm - t : t - tm, db = tb > t ? tb - t : t - tb;
    if (da <= dm && da <= db) return imin;
    if (dm <= da && dm <= db) return imid;
    return imax;
}

// The 20 consecutive candidates of :500-530: back from `found`, topped up forward when fewer than 20 lie behind.  [lo, hi)
#if defined(__CUDACC__)
__host__ __device__
#endif
inline void deform_window(int found, int n, int* lo, int* hi)
{
    int l = found - (DEFORM_LOOKBACK - 1); if (l < 0) l = 0;
    int h = l + DEFORM_LOOKBACK; if (h > n) h = n;
    *lo = l; *hi = h;
}

// One candidate (distance d, node j; j ascending over the window) into the k + 1 nearest, bd / bi ordered by (distance, id) and
// started at (+inf, INT_MAX).  A NaN distance (a non-finite vertex) counts as +inf, and +inf candidates are still taken in id order,
// so after a window of at least k + 1 nodes every slot holds a node of that window.
#if defined(__CUDACC__)
__host__ __device__
#endif
inline void deform_insert(float d, int j, float* bd, int* bi)
{
    if (d != d) d = INFINITY;
    if (!(d < bd[DEFORM_K] || (d == bd[DEFORM_K] && j < bi[DEFORM_K]))) return;
    float cd = d; int ci = j;
    for (int q = 0; q <= DEFORM_K; ++q)
        if (cd < bd[q] || (cd == bd[q] && ci < bi[q])) { const float td = bd[q]; const int ti = bi[q]; bd[q] = cd; bi[q] = ci; cd = td; ci = ti; }
}

// Index of the first value that is not finite (NaN or +-inf) among n, or -1.  Constraint sources and targets, corrected positions and
// node positions come from the caller (a failed PnP inlier can be NaN); one that is not finite is rejected before any kernel runs.
template <class T> inline long deform_first_non_finite(const T* v, size_t n)
{
    for (size_t i = 0; i < n; ++i) if (!std::isfinite(v[i])) return (long)i;
    return -1;
}

// addCameraLoop (:237-276): every corrected camera pose contributes the tracked camera position at its timestamp (the source, a vertex
// with that time) and its corrected position (the target).  Only positions are used, as in the reference.  pose timestamps / positions
// come from the dense pose graph; a timestamp that occurs twice there maps to its last record (the reference's std::map cameraPoseMap).
// Returns the index of the first corrected timestamp that is not in the graph, or -1 when all were found.
struct DeformConstraint { uint64_t time; float src[3]; double dst[3]; };
inline long deform_pose_constraints(const uint64_t* graph_times, const float* graph_pos, size_t n_graph,
                                    const uint64_t* corr_times, const double* corr_pos, size_t n_corr, std::vector<DeformConstraint>& out)
{
    std::unordered_map<uint64_t, size_t> at;
    at.reserve(n_graph * 2 + 1);
    for (size_t i = 0; i < n_graph; ++i) at[graph_times[i]] = i;
    for (size_t i = 0; i < n_corr; ++i) {
        auto it = at.find(corr_times[i]);
        if (it == at.end()) return (long)i;
        DeformConstraint c; c.time = corr_times[i];
        for (int d = 0; d < 3; ++d) { c.src[d] = graph_pos[3 * it->second + d]; c.dst[d] = corr_pos[3 * i + d]; }
        out.push_back(c);
    }
    return -1;
}

} // namespace kt
