// Host build of kintinuous_b200/csrc/kt_deform.hpp for tests/test_deform_oracle.py.
#include "kt_deform.hpp"
#include <cmath>
#include <cstring>
extern "C" {
int kth_sample_nodes(const float* pos, size_t n, float pose_dist, int* out)
{
    const std::vector<int> t = kt::deform_sample_nodes(pos, n, pose_dist);
    std::memcpy(out, t.data(), t.size() * sizeof(int));
    return (int)t.size();
}
int kth_connect_seq(int n, int* off, int* out)
{
    std::vector<int> o, nb; kt::deform_connect_seq(n, kt::DEFORM_K, o, nb);
    std::memcpy(off, o.data(), o.size() * sizeof(int)); std::memcpy(out, nb.data(), nb.size() * sizeof(int));
    return (int)nb.size();
}
// the k + 1 nearest of a window [lo, lo + n) of candidate distances, as deform_weight_kernel keeps them
void kth_select(const float* d, int lo, int n, float* bd, int* bi)
{
    for (int q = 0; q <= kt::DEFORM_K; ++q) { bd[q] = INFINITY; bi[q] = 2147483647; }
    for (int j = 0; j < n; ++j) kt::deform_insert(d[j], lo + j, bd, bi);
}
long kth_first_non_finite_f(const float* v, size_t n) { return kt::deform_first_non_finite(v, n); }
long kth_first_non_finite_d(const double* v, size_t n) { return kt::deform_first_non_finite(v, n); }
int kth_nearest_node(const uint64_t* times, int n, uint64_t t) { return kt::deform_nearest_node(times, n, t); }
long kth_pose_constraints(const uint64_t* gt, const float* gp, size_t ng, const uint64_t* ct, const double* cp, size_t nc, float* src, double* dst)
{
    std::vector<kt::DeformConstraint> c;
    const long miss = kt::deform_pose_constraints(gt, gp, ng, ct, cp, nc, c);
    for (size_t i = 0; i < c.size(); ++i) for (int e = 0; e < 3; ++e) { src[3 * i + e] = c[i].src[e]; dst[3 * i + e] = c[i].dst[e]; }
    return miss;
}
}
