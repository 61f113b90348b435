// Host build of kintinuous_b200/csrc/kt_place.hpp for tests/test_place_oracle.py.
#include "kt_place.hpp"
#include <cstring>
extern "C" {
int kth_is_keyframe(const float* Rc, const float* Rl, const float* gc, const float* gl) { return kt::place_is_keyframe(Rc, Rl, gc, gl) ? 1 : 0; }
double kth_motion(const float* Rc, const float* Rl, const float* gc, const float* gl) { return kt::place_motion(Rc, Rl, gc, gl); }
int kth_select_candidate(const int* passes, int query, int exclude_recent, int min_passes) { return kt::place_select_candidate(passes, query, exclude_recent, min_passes); }
int kth_lookup_3d(float x, float y, const uint16_t* depth, int rows, int cols, const float* intr4, float* xyz) { return kt::place_lookup_3d(x, y, depth, rows, cols, intr4, xyz) ? 1 : 0; }
int kth_unique_matches(const int* best, const float* d1, const unsigned char* pass, int n_old, int n_new, int* old_idx, int* new_idx)
{
    std::vector<int> a, b;
    kt::place_unique_matches(best, d1, pass, n_old, n_new, a, b);
    if (!a.empty()) { std::memcpy(old_idx, a.data(), a.size() * sizeof(int)); std::memcpy(new_idx, b.data(), b.size() * sizeof(int)); }
    return (int)a.size();
}
int kth_match_3d(const int* best, const float* d1, const unsigned char* pass, int n_old, int n_new, const float* xyz_old, const float* xyz_new,
                 int* old_idx, int* new_idx)
{
    std::vector<int> a, b;
    kt::place_match_3d(best, d1, pass, n_old, n_new, xyz_old, xyz_new, a, b);
    if (!a.empty()) { std::memcpy(old_idx, a.data(), a.size() * sizeof(int)); std::memcpy(new_idx, b.data(), b.size() * sizeof(int)); }
    return (int)a.size();
}
int kth_project_inliers(const float* kp_new, const float* kp_old, const unsigned char* inl, int n, const uint16_t* dn, const uint16_t* dold, int rows, int cols,
                        const float* intr4, float* out_new, float* out_old)
{
    std::vector<float> a, b;
    kt::place_project_inliers(kp_new, kp_old, inl, n, dn, dold, rows, cols, intr4, a, b);
    if (!a.empty()) { std::memcpy(out_new, a.data(), a.size() * sizeof(float)); std::memcpy(out_old, b.data(), b.size() * sizeof(float)); }
    return (int)(a.size() / 3);
}
int kth_throttled(uint64_t last, uint64_t now, double s) { return kt::place_throttled(last, now, s) ? 1 : 0; }
}
