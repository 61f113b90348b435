// kintinuous_b200 -- the CUDA-free decisions of place recognition (kt_detect_loops, kt_place.cu), CPU-tested through tests/cpp/place_host.cpp
// (tests/test_place_oracle.py).
//
// Stands in for (reference, src/): the keyframe rule of KintinuousTracker::processFrame (frontend/KintinuousTracker.cpp:605-624,
// 706-718), the candidate that DLoopDetector returns (here: exhaustive ratio-test retrieval, kt_place.cu), Surf3DTools::surfMatch3D's
// pairing and 3-D lookup (backend/Surf3DTools.h:105-274) and DepthCamera::projectInlierMatches (backend/DepthCamera.cpp:66-93).
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

namespace kt {

// (|rodrigues(Rcurr^-1 R_last)| + |g_curr - g_last|) / 2 >= movement (KintinuousTracker.cpp:607-611, alpha = 1, movement 0.15).
// R row-major, g = currentGlobalCamera.  The angle of a rotation is |rodrigues(R)|; for R^T R_last it is acos((tr - 1) / 2), taken
// through atan2 of the skew part so that it stays exact near 0 and pi.
inline double place_motion(const float* R_curr, const float* R_last, const float* g_curr, const float* g_last)
{
    double M[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double s = 0;
            for (int k = 0; k < 3; ++k) s += (double)R_curr[k * 3 + i] * (double)R_last[k * 3 + j];     // Rcurr^T R_last = Rcurr^-1 R_last
            M[i * 3 + j] = s;
        }
    const double sx = M[7] - M[5], sy = M[2] - M[6], sz = M[3] - M[1];
    const double ang = std::atan2(0.5 * std::sqrt(sx * sx + sy * sy + sz * sz), 0.5 * (M[0] + M[4] + M[8] - 1.0));
    double t = 0;
    for (int e = 0; e < 3; ++e) { const double d = (double)g_curr[e] - (double)g_last[e]; t += d * d; }
    return 0.5 * (ang + std::sqrt(t));
}
inline bool place_is_keyframe(const float* R_curr, const float* R_last, const float* g_curr, const float* g_last, double movement = 0.15)
{
    return place_motion(R_curr, R_last, g_curr, g_last) >= movement;
}

// The candidate of keyframe `query` from the pass counts of every keyframe before it: the keyframe with the most passes among those at
// least exclude_recent keyframes older (index <= query - exclude_recent), ties to the older one, and at least min_passes of them.
// -1: no candidate.
inline int place_select_candidate(const int* passes, int query, int exclude_recent, int min_passes)
{
    int best = -1, bp = 0;
    for (int k = 0; k <= query - exclude_recent; ++k)
        if (passes[k] > bp) { bp = passes[k]; best = k; }        // strict: the older keyframe keeps a tie
    return bp >= min_passes ? best : -1;
}

// (x, y) of a keypoint -> the pixel within +-0.5 px, STRICT (Surf3DTools.h:142-160: a coordinate that is exactly half-way between two
// pixels has none), then depth != 0 and z < 10 m (Surf3DTools.h:82 drops |z - 10| < FLT_EPSILON and |z| > 10: for depths in whole
// millimetres that is z < 10); back-projection with the depth intrinsics.  false: no 3-D point.
inline bool place_lookup_pixel(float x, float y, int rows, int cols, int* u, int* v)
{
    const int ui = (int)std::floor(x + 0.5f), vi = (int)std::floor(y + 0.5f);
    if (!(std::fabs((float)ui - x) < 0.5f && std::fabs((float)vi - y) < 0.5f)) return false;
    if (ui < 0 || vi < 0 || ui >= cols || vi >= rows) return false;
    *u = ui; *v = vi;
    return true;
}
inline bool place_lookup_3d(float x, float y, const uint16_t* depth, int rows, int cols, const float* intr4, float* xyz)
{
    int u, v;
    if (!place_lookup_pixel(x, y, rows, cols, &u, &v)) return false;
    const uint16_t d = depth[(size_t)v * cols + u];
    if (d == 0) return false;
    const float z = (float)d / 1000.f;
    if (!(z < 10.f)) return false;
    xyz[0] = z * ((float)u - intr4[2]) / intr4[0]; xyz[1] = z * ((float)v - intr4[3]) / intr4[1]; xyz[2] = z;
    return true;
}

// One match per new feature (quirk R8 in DESIGN's table): every old feature (row) that passes the ratio test names its nearest
// new feature best[i] at squared distance d1[i]; a new feature named by several old ones keeps the nearest, ties to the lower old index
// (surfMatch3D keeps the last one, and never an old feature 0).  Output: (old, new) pairs in ascending new index.
inline void place_unique_matches(const int* best, const float* d1, const unsigned char* pass, int n_old, int n_new, std::vector<int>& old_idx,
                                 std::vector<int>& new_idx)
{
    std::vector<int> owner((size_t)(n_new > 0 ? n_new : 0), -1);
    for (int i = 0; i < n_old; ++i) {
        if (!pass[i] || best[i] < 0 || best[i] >= n_new) continue;
        int& o = owner[(size_t)best[i]];
        if (o < 0 || d1[i] < d1[o]) o = i;
    }
    old_idx.clear(); new_idx.clear();
    for (int j = 0; j < n_new; ++j) if (owner[(size_t)j] >= 0) { old_idx.push_back(owner[(size_t)j]); new_idx.push_back(j); }
}

// Surf3DTools::surfMatch3D (Surf3DTools.h:105-176) in the reference's order: the ratio test over ALL features of both keyframes (its
// result: best / d1 / pass per old feature), one match per new feature (place_unique_matches), THEN the pairs whose old or new keypoint
// has no 3-D point are dropped -- a new feature whose chosen old feature has no depth gets no match.  xyz_*: 3 floats per feature, NaN
// (z != z) without a point.
inline void place_match_3d(const int* best, const float* d1, const unsigned char* pass, int n_old, int n_new, const float* xyz_old, const float* xyz_new,
                           std::vector<int>& old_idx, std::vector<int>& new_idx)
{
    std::vector<int> oi, ni;
    place_unique_matches(best, d1, pass, n_old, n_new, oi, ni);
    old_idx.clear(); new_idx.clear();
    for (size_t k = 0; k < oi.size(); ++k) {
        const float zo = xyz_old[(size_t)oi[k] * 3 + 2], zn = xyz_new[(size_t)ni[k] * 3 + 2];
        if (zo == zo && zn == zn) { old_idx.push_back(oi[k]); new_idx.push_back(ni[k]); }
    }
}

// DepthCamera::projectInlierMatches (DepthCamera.cpp:66-93): an inlier's keypoints are back-projected at their TRUNCATED pixel
// coordinates ((int)x, (int)y) with the depth of that pixel; a pair where either depth is 0 is dropped.  kp_*: x, y per match; out:
// xyz triples appended.
inline void place_project_inliers(const float* kp_new, const float* kp_old, const unsigned char* inlier, int n, const uint16_t* depth_new,
                                  const uint16_t* depth_old, int rows, int cols, const float* intr4, std::vector<float>& in_new, std::vector<float>& in_old)
{
    in_new.clear(); in_old.clear();
    for (int i = 0; i < n; ++i) {
        if (!inlier[i]) continue;
        const int u1 = (int)kp_new[2 * i], v1 = (int)kp_new[2 * i + 1], u2 = (int)kp_old[2 * i], v2 = (int)kp_old[2 * i + 1];
        if (u1 < 0 || v1 < 0 || u1 >= cols || v1 >= rows || u2 < 0 || v2 < 0 || u2 >= cols || v2 >= rows) continue;
        const float z1 = (float)depth_new[(size_t)v1 * cols + u1] / 1000.f, z2 = (float)depth_old[(size_t)v2 * cols + u2] / 1000.f;
        if (z1 == 0.f || z2 == 0.f) continue;
        const double ifx = 1.0 / (double)intr4[0], ify = 1.0 / (double)intr4[1];
        in_new.push_back((float)(z1 * ((double)u1 - intr4[2]) * ifx)); in_new.push_back((float)(z1 * ((double)v1 - intr4[3]) * ify)); in_new.push_back(z1);
        in_old.push_back((float)(z2 * ((double)u2 - intr4[2]) * ifx)); in_old.push_back((float)(z2 * ((double)v2 - intr4[3]) * ify)); in_old.push_back(z2);
    }
}

// The -lt throttle (PlaceRecognition.cpp:118-123) on frame timestamps: a keyframe within throttle_us of the last loop found is not tried.
inline bool place_throttled(uint64_t last_loop, uint64_t now, double throttle_s)
{
    return last_loop > 0 && now >= last_loop && (double)(now - last_loop) <= throttle_s * 1e6;
}

} // namespace kt
