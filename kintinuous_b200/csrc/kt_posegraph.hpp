// kintinuous_b200 -- the dense pose graph record and the <saveFile>.poses trajectory line, CUDA-free (host logic; CPU-tested through
// tests/cpp/posegraph_host.cpp).
//
// Replaces (reference, src/frontend/):
//   KintinuousTracker::DensePose / densePoseGraph / latestDensePoseId        KintinuousTracker.h:151-172, .cpp:529-536, :901-909
//   KintinuousTracker::outputPose                                           KintinuousTracker.cpp:199-218 (called per frame, :911-914)
// outputPose writes  "<utime / 1e6, fixed, 6 decimals> gx gy gz qx qy qz qw\n"  with the floats in the stream's default format (%g,
// 6 significant digits) and the quaternion from Eigen::Quaternionf(Rcurr).  Eigen is a third-party dependency that is not under
// the reference checkout: its matrix -> quaternion conversion (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl<Other,3,3>, the
// same in every 3.x release) is restated below in float.  The reference re-opens, appends and closes the file on EVERY frame
// (SURVEY.md Q14); here the file stays open for the life of the context and every line is flushed.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>

namespace kt {

// Eigen::Quaternionf(Matrix3f): returns x, y, z, w
inline void quaternion_from_rotation(const float* m /* row-major 3x3 */, float* q4)
{
    float t = m[0] + m[4] + m[8];
    float w, x, y, z;
    if (t > 0.0f) {
        t = std::sqrt(t + 1.0f);
        w = 0.5f * t;
        t = 0.5f / t;
        x = (m[2 * 3 + 1] - m[1 * 3 + 2]) * t;
        y = (m[0 * 3 + 2] - m[2 * 3 + 0]) * t;
        z = (m[1 * 3 + 0] - m[0 * 3 + 1]) * t;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 3 + i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0f);
        float q[3];
        q[i] = 0.5f * t;
        t = 0.5f / t;
        w = (m[k * 3 + j] - m[j * 3 + k]) * t;
        q[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
        q[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
        x = q[0]; y = q[1]; z = q[2];
    }
    q4[0] = x; q4[1] = y; q4[2] = z; q4[3] = w;
}

// One line of <saveFile>.poses exactly as outputPose streams it.  Returns the line's length (without the terminating 0), or -1 if it
// does not fit.
inline int format_pose_line(uint64_t timestamp, const float* global_t3, const float* R9, char* buf, size_t cap)
{
    float q[4];
    quaternion_from_rotation(R9, q);
    // std::setprecision(6) << std::fixed on the double timestamp; operator<<(float) afterwards on a fresh stream = %g
    const int n = std::snprintf(buf, cap, "%.6f %g %g %g %g %g %g %g\n", (double)timestamp / 1000000.0,
                                (double)global_t3[0], (double)global_t3[1], (double)global_t3[2], (double)q[0], (double)q[1], (double)q[2], (double)q[3]);
    return (n < 0 || (size_t)n >= cap) ? -1 : n;
}

} // namespace kt
