// Host build of kintinuous_b200/csrc/kt_pgo.hpp for tests/test_pgo_oracle.py.
#include "kt_pgo.hpp"
#include <cstring>
extern "C" {
void kth_odometry_z(const float* prev, const float* curr, double* z) { kt::pgo_odometry_z(prev, curr, z); }
void kth_loop_z(const double* C, double* z) { kt::pgo_loop_z(C, z); }
int kth_check_constraint(const double* C) { return kt::pgo_check_constraint(C); }
int kth_select_nodes(const float* pos, const unsigned char* flagged, size_t n, float spacing, int* out)
{
    const std::vector<int> t = kt::pgo_select_nodes(pos, flagged, n, spacing);
    std::memcpy(out, t.data(), t.size() * sizeof(int));
    return (int)t.size();
}
void kth_pose_to_isam(const float* P, double* X) { kt::pgo_pose_to_isam(P, X); }
void kth_pose_from_isam(const double* X, double* P) { kt::pgo_pose_from_isam(X, P); }
double kth_wrap(double a) { return kt::pgo_wrap(a); }
void kth_ypr(const double* R, double* v) { kt::pgo_ypr(R, v); }
void kth_rot(const double* v, double* R) { kt::pgo_rot(v, R); }
// levels of the plan and the loop endpoints at the top level; sizes[l] = nodes of level l
int kth_plan(int n, int L, const int* li, const int* lj, int* sizes, int max_levels, int* top_i, int* top_j)
{
    const kt::PgoPlan p = kt::pgo_plan(n, std::vector<int>(li, li + L), std::vector<int>(lj, lj + L));
    for (int l = 0; l < (int)p.n.size() && l < max_levels; ++l) sizes[l] = p.n[l];
    for (int l = 0; l < L; ++l) { top_i[l] = p.loop_i[l]; top_j[l] = p.loop_j[l]; }
    return (int)p.n.size();
}
}
