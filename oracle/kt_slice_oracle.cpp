// TEST INFRASTRUCTURE ONLY (oracle/): never linked into, imported by or executed from the product path (kintinuous_b200/).
//
// CPU restatement of the post-processing CloudSliceProcessor applies to every slice the tracker hands out
// (reference: src/backend/CloudSliceProcessor.cpp:97-151):
//     1. weight cull        keep points with alpha >= ConfigArgs::weightCull (-cw, default 8)            :104-121
//     2. pcl::VoxelGrid     leaf = max voxel edge, one centroid per occupied leaf                        :126-148
//     3. pcl::NormalEstimation, KdTree, setKSearch(20)                                                   :150-160
//     4. pcl::concatenateFields -> PointXYZRGBNormal                                                     :162
// Steps 2 and 3 live in a third-party dependency that is NOT under the reference checkout: PCL, "find_package(PCL 1.7)" (src/CMakeLists.txt:52),
// installed by build.sh from the 14.04 PPA = PCL 1.7.2.  This file restates the published algorithms of PCL 1.7.2:
//     filters/include/pcl/filters/impl/voxel_grid.hpp        VoxelGrid<PointT>::applyFilter
//     common/include/pcl/common/impl/centroid.hpp            computeMeanAndCovarianceMatrix (single pass, float accumulators)
//     common/include/pcl/common/impl/eigen.hpp               computeRoots / computeRoots2 / eigen33 (smallest eigenvalue + eigenvector)
//     features/include/pcl/features/normal_3d.h              computePointNormal, solvePlaneParameters, flipNormalTowardsViewpoint (vp = 0,0,0)
// PINNING STATUS: parity unpinned against PCL itself (PCL does not exist in this image and the reference ships no fixtures for this step).
// The restatement is pinned piecewise instead (tests/test_slice_oracle.py): leaf assignment / centroids against an independent numpy
// statement, the analytic eigen solver against numpy.linalg.eigh, the neighbour search against brute force.
// Unspecified in PCL and fixed here: the order of points inside a leaf (std::sort is not stable; here: input order) and the order of
// equidistant neighbours (FLANN; here: by index).  Both only permute float additions.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>
#include <algorithm>
#include <limits>

namespace {

struct PointIn { float x, y, z, pad0; uint8_t b, g, r, a; uint8_t pad1[12]; };                               // pcl::PointXYZRGB (32 B)
struct PointOut { float x, y, z, pad0; float nx, ny, nz, pad1; uint8_t b, g, r, a; float curvature; float pad2[2]; };   // pcl::PointXYZRGBNormal (48 B)
static_assert(sizeof(PointIn) == 32 && sizeof(PointOut) == 48, "PCL point layouts");

// ---- pcl/common/impl/eigen.hpp (1.7.2), Scalar = float ----
void compute_roots2(float b, float c, float* roots)
{
    roots[0] = 0.f;
    float d = b * b - 4.0f * c;
    if (d < 0.0f) d = 0.0f;
    const float sd = std::sqrt(d);
    roots[2] = 0.5f * (b + sd);
    roots[1] = 0.5f * (b - sd);
}

void compute_roots(const float* m /* 3x3 symmetric, row-major */, float* roots)
{
    const float c0 = m[0] * m[4] * m[8] + 2.f * m[1] * m[2] * m[5] - m[0] * m[5] * m[5] - m[4] * m[2] * m[2] - m[8] * m[1] * m[1];
    const float c1 = m[0] * m[4] - m[1] * m[1] + m[0] * m[8] - m[2] * m[2] + m[4] * m[8] - m[5] * m[5];
    const float c2 = m[0] + m[4] + m[8];
    if (std::fabs(c0) < std::numeric_limits<float>::epsilon()) { compute_roots2(c2, c1, roots); return; }
    const float s_inv3 = 1.0f / 3.0f, s_sqrt3 = std::sqrt(3.0f);
    const float c2_over_3 = c2 * s_inv3;
    float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
    if (a_over_3 > 0.f) a_over_3 = 0.f;
    const float half_b = 0.5f * (c0 + c2_over_3 * (2.f * c2_over_3 * c2_over_3 - c1));
    float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
    if (q > 0.f) q = 0.f;
    const float rho = std::sqrt(-a_over_3);
    const float theta = std::atan2(std::sqrt(-q), half_b) * s_inv3;
    const float cos_theta = std::cos(theta), sin_theta = std::sin(theta);
    roots[0] = c2_over_3 + 2.f * rho * cos_theta;
    roots[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
    roots[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
    if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]);
    if (roots[1] >= roots[2]) { std::swap(roots[1], roots[2]); if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]); }
    if (roots[0] <= 0.f) compute_roots2(c2, c1, roots);          // "eigenvalue for symmetric positive semi-definite matrix can not be negative"
}

void eigen33_smallest(const float* mat, float* eigenvalue, float* eigenvector)
{
    float scale = 0.f;
    for (int i = 0; i < 9; ++i) scale = std::max(scale, std::fabs(mat[i]));
    if (scale <= std::numeric_limits<float>::min()) scale = 1.0f;
    float s[9];
    for (int i = 0; i < 9; ++i) s[i] = mat[i] / scale;
    float roots[3];
    compute_roots(s, roots);
    *eigenvalue = roots[0] * scale;
    s[0] -= roots[0]; s[4] -= roots[0]; s[8] -= roots[0];
    const float* r0 = s; const float* r1 = s + 3; const float* r2 = s + 6;
    const float v1[3] = {r0[1] * r1[2] - r0[2] * r1[1], r0[2] * r1[0] - r0[0] * r1[2], r0[0] * r1[1] - r0[1] * r1[0]};
    const float v2[3] = {r0[1] * r2[2] - r0[2] * r2[1], r0[2] * r2[0] - r0[0] * r2[2], r0[0] * r2[1] - r0[1] * r2[0]};
    const float v3[3] = {r1[1] * r2[2] - r1[2] * r2[1], r1[2] * r2[0] - r1[0] * r2[2], r1[0] * r2[1] - r1[1] * r2[0]};
    const float l1 = v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2];
    const float l2 = v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2];
    const float l3 = v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2];
    const float* v; float l;
    if (l1 >= l2 && l1 >= l3) { v = v1; l = l1; } else if (l2 >= l1 && l2 >= l3) { v = v2; l = l2; } else { v = v3; l = l3; }
    const float inv = std::sqrt(l);
    for (int i = 0; i < 3; ++i) eigenvector[i] = v[i] / inv;
}

// ---- pcl/features/normal_3d.h: computePointNormal over the given neighbours, then flipNormalTowardsViewpoint(vp = origin) ----
void point_normal(const std::vector<PointOut>& cloud, const int* nn, int k, const PointOut& query, float* n4)
{
    const float nan = std::numeric_limits<float>::quiet_NaN();
    if (k < 3) { n4[0] = n4[1] = n4[2] = n4[3] = nan; return; }
    float accu[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};                     // centroid.hpp: single pass, float accumulators
    for (int i = 0; i < k; ++i) {
        const PointOut& p = cloud[nn[i]];
        accu[0] += p.x * p.x; accu[1] += p.x * p.y; accu[2] += p.x * p.z;
        accu[3] += p.y * p.y; accu[4] += p.y * p.z; accu[5] += p.z * p.z;
        accu[6] += p.x; accu[7] += p.y; accu[8] += p.z;
    }
    for (int i = 0; i < 9; ++i) accu[i] /= (float)k;
    float cov[9];
    cov[0] = accu[0] - accu[6] * accu[6]; cov[1] = accu[1] - accu[6] * accu[7]; cov[2] = accu[2] - accu[6] * accu[8];
    cov[4] = accu[3] - accu[7] * accu[7]; cov[5] = accu[4] - accu[7] * accu[8]; cov[8] = accu[5] - accu[8] * accu[8];
    cov[3] = cov[1]; cov[6] = cov[2]; cov[7] = cov[5];
    float ev, vec[3];
    eigen33_smallest(cov, &ev, vec);
    const float eig_sum = cov[0] + cov[4] + cov[8];
    float curvature = eig_sum != 0 ? std::fabs(ev / eig_sum) : 0.f;
    // flipNormalTowardsViewpoint(point, 0, 0, 0, nx, ny, nz)
    const float vx = 0.f - query.x, vy = 0.f - query.y, vz = 0.f - query.z;
    const float cos_theta = vx * vec[0] + vy * vec[1] + vz * vec[2];
    if (cos_theta < 0) { vec[0] *= -1; vec[1] *= -1; vec[2] *= -1; }
    n4[0] = vec[0]; n4[1] = vec[1]; n4[2] = vec[2]; n4[3] = curvature;
}

} // namespace

extern "C" {

// Exposed for piecewise pinning (tests/test_slice_oracle.py)
void ktslice_eigen33(const float* cov9, float* eigenvalue, float* eigenvector3) { eigen33_smallest(cov9, eigenvalue, eigenvector3); }

// CloudSliceProcessor.cpp:104-121 -- returns the number of kept points (written to out, input order)
size_t ktslice_weight_cull(const void* in, size_t n, int weight_cull, void* out)
{
    const PointIn* p = (const PointIn*)in; PointIn* o = (PointIn*)out;
    size_t m = 0;
    for (size_t i = 0; i < n; ++i) if (weight_cull <= 0 || p[i].a >= weight_cull) o[m++] = p[i];
    return m;
}

// pcl::VoxelGrid<PointXYZRGB>::applyFilter (PCL 1.7.2), downsample_all_data = true, min_points_per_voxel = 0, no filter field.
// Returns the number of output points (leaf order); writes at most cap.  leaf_index_out (optional): per output point the PCL leaf index
// and min_b (3 ints appended at [cap*1 ...] is NOT done; min_b is returned through min_b3).
size_t ktslice_voxel_grid(const void* in, size_t n, float leaf, void* out, size_t cap, int* min_b3, int* div_b3)
{
    const PointIn* p = (const PointIn*)in; PointIn* o = (PointIn*)out;
    if (n == 0) return 0;
    float mn[3] = {std::numeric_limits<float>::max(), std::numeric_limits<float>::max(), std::numeric_limits<float>::max()}, mx[3] = {-mn[0], -mn[0], -mn[0]};
    for (size_t i = 0; i < n; ++i) {                                                                            // getMinMax3D
        mn[0] = std::min(mn[0], p[i].x); mn[1] = std::min(mn[1], p[i].y); mn[2] = std::min(mn[2], p[i].z);
        mx[0] = std::max(mx[0], p[i].x); mx[1] = std::max(mx[1], p[i].y); mx[2] = std::max(mx[2], p[i].z);
    }
    const float inv = 1.0f / leaf;                                                                              // inverse_leaf_size_
    const int64_t dx = (int64_t)((mx[0] - mn[0]) * inv) + 1, dy = (int64_t)((mx[1] - mn[1]) * inv) + 1, dz = (int64_t)((mx[2] - mn[2]) * inv) + 1;
    if (dx * dy * dz > (int64_t)std::numeric_limits<int32_t>::max()) {                                          // "Leaf size is too small ... Integer indices would overflow": output = input
        const size_t m = std::min(n, cap);
        memcpy(o, p, m * sizeof(PointIn));
        if (min_b3) min_b3[0] = min_b3[1] = min_b3[2] = 0;
        if (div_b3) div_b3[0] = div_b3[1] = div_b3[2] = 0;
        return m;
    }
    int min_b[3], max_b[3], div_b[3];
    for (int i = 0; i < 3; ++i) { min_b[i] = (int)std::floor(mn[i] * inv); max_b[i] = (int)std::floor(mx[i] * inv); div_b[i] = max_b[i] - min_b[i] + 1; }
    const int mul[3] = {1, div_b[0], div_b[0] * div_b[1]};
    if (min_b3) for (int i = 0; i < 3; ++i) min_b3[i] = min_b[i];
    if (div_b3) for (int i = 0; i < 3; ++i) div_b3[i] = div_b[i];
    std::vector<std::pair<int, uint32_t> > iv(n);
    for (size_t i = 0; i < n; ++i) {
        const int i0 = (int)(std::floor(p[i].x * inv) - (float)min_b[0]);
        const int i1 = (int)(std::floor(p[i].y * inv) - (float)min_b[1]);
        const int i2 = (int)(std::floor(p[i].z * inv) - (float)min_b[2]);
        iv[i] = std::make_pair(i0 * mul[0] + i1 * mul[1] + i2 * mul[2], (uint32_t)i);
    }
    std::stable_sort(iv.begin(), iv.end(), [](const std::pair<int, uint32_t>& a, const std::pair<int, uint32_t>& b) { return a.first < b.first; });
    size_t m = 0;
    for (size_t first = 0; first < n;) {
        size_t last = first + 1;
        while (last < n && iv[last].first == iv[first].first) ++last;
        float c[6] = {0, 0, 0, 0, 0, 0};                                                                        // Eigen::VectorXf centroid: x, y, z, (rgb as float: ignored), r, g, b
        for (size_t j = first; j < last; ++j) {
            const PointIn& q = p[iv[j].second];
            c[0] += q.x; c[1] += q.y; c[2] += q.z; c[3] += (float)q.r; c[4] += (float)q.g; c[5] += (float)q.b;
        }
        const float cnt = (float)(last - first);
        for (int k = 0; k < 6; ++k) c[k] /= cnt;
        if (m < cap) {
            PointIn r; memset(&r, 0, sizeof(r));
            r.x = c[0]; r.y = c[1]; r.z = c[2];
            r.pad0 = 1.0f;                                                                                     // PointXYZRGB default data[3]
            const int rgb = ((int)c[3]) << 16 | ((int)c[4]) << 8 | ((int)c[5]);                                // alpha byte ends up 0
            r.r = (uint8_t)(rgb >> 16); r.g = (uint8_t)(rgb >> 8); r.b = (uint8_t)rgb; r.a = 0;
            o[m] = r;
        }
        ++m;
        first = last;
    }
    return std::min(m, cap);
}

// pcl::NormalEstimation::computeFeature with setKSearch(k) over the cloud itself + concatenateFields.  Exact k nearest neighbours
// (including the query point) through a uniform grid of cell `cell`; neighbours ordered by (distance, index).
void ktslice_normals(const void* in, size_t n, int k, float cell, void* out48)
{
    const PointIn* p = (const PointIn*)in; PointOut* o = (PointOut*)out48;
    std::vector<PointOut> cloud(n);
    for (size_t i = 0; i < n; ++i) { PointOut q; memset(&q, 0, sizeof(q)); q.x = p[i].x; q.y = p[i].y; q.z = p[i].z; q.pad0 = 1.0f; q.b = p[i].b; q.g = p[i].g; q.r = p[i].r; q.a = p[i].a; cloud[i] = q; }
    if (n == 0) return;
    // grid
    float mn[3] = {p[0].x, p[0].y, p[0].z}, mx[3] = {p[0].x, p[0].y, p[0].z};
    for (size_t i = 1; i < n; ++i) { mn[0] = std::min(mn[0], p[i].x); mn[1] = std::min(mn[1], p[i].y); mn[2] = std::min(mn[2], p[i].z); mx[0] = std::max(mx[0], p[i].x); mx[1] = std::max(mx[1], p[i].y); mx[2] = std::max(mx[2], p[i].z); }
    const double inv = 1.0 / cell;
    int dim[3];
    for (int a = 0; a < 3; ++a) dim[a] = (int)std::floor((mx[a] - mn[a]) * inv) + 1;
    auto cidx = [&](const PointIn& q, int* c) { c[0] = std::min(dim[0] - 1, std::max(0, (int)std::floor((q.x - mn[0]) * inv))); c[1] = std::min(dim[1] - 1, std::max(0, (int)std::floor((q.y - mn[1]) * inv))); c[2] = std::min(dim[2] - 1, std::max(0, (int)std::floor((q.z - mn[2]) * inv))); };
    const size_t ncell = (size_t)dim[0] * dim[1] * dim[2];
    std::vector<uint32_t> start(ncell + 1, 0), order(n);
    std::vector<size_t> lin(n);
    for (size_t i = 0; i < n; ++i) { int c[3]; cidx(p[i], c); lin[i] = ((size_t)c[2] * dim[1] + c[1]) * dim[0] + c[0]; ++start[lin[i] + 1]; }
    for (size_t i = 0; i < ncell; ++i) start[i + 1] += start[i];
    { std::vector<uint32_t> fill(start.begin(), start.end() - 1); for (size_t i = 0; i < n; ++i) order[fill[lin[i]]++] = (uint32_t)i; }
    const int kk = (int)std::min<size_t>((size_t)k, n);
    std::vector<std::pair<float, uint32_t> > cand;
    std::vector<int> nn(kk);
    const int rmax = std::max(dim[0], std::max(dim[1], dim[2]));
    for (size_t i = 0; i < n; ++i) {
        int c[3]; cidx(p[i], c);
        for (int r = 1;; ++r) {
            cand.clear();
            for (int z = std::max(0, c[2] - r); z <= std::min(dim[2] - 1, c[2] + r); ++z)
                for (int y = std::max(0, c[1] - r); y <= std::min(dim[1] - 1, c[1] + r); ++y)
                    for (int x = std::max(0, c[0] - r); x <= std::min(dim[0] - 1, c[0] + r); ++x) {
                        const size_t l = ((size_t)z * dim[1] + y) * dim[0] + x;
                        for (uint32_t s = start[l]; s < start[l + 1]; ++s) {
                            const PointIn& q = p[order[s]];
                            const float dx = q.x - p[i].x, dy = q.y - p[i].y, dz = q.z - p[i].z;
                            cand.push_back(std::make_pair(dx * dx + dy * dy + dz * dz, order[s]));
                        }
                    }
            if ((int)cand.size() >= kk) {
                std::sort(cand.begin(), cand.end());
                // every point outside the cube of +-r cells is farther than r * cell from the query along some axis
                const double reach = (double)r * cell;
                if (r >= rmax || (double)cand[kk - 1].first <= reach * reach) break;
            } else if (r >= rmax) { std::sort(cand.begin(), cand.end()); break; }
        }
        const int got = (int)std::min<size_t>(cand.size(), (size_t)kk);
        for (int j = 0; j < got; ++j) nn[j] = (int)cand[j].second;
        float n4[4];
        point_normal(cloud, nn.data(), got, cloud[i], n4);
        PointOut q = cloud[i];
        q.nx = n4[0]; q.ny = n4[1]; q.nz = n4[2]; q.pad1 = 0.f; q.curvature = n4[3];
        o[i] = q;
    }
}

// The whole chain of CloudSliceProcessor.cpp:97-162 on one slice.  Returns the number of processed points (<= cap).
size_t ktslice_process(const void* in, size_t n, int weight_cull, float leaf, int k, void* out48, size_t cap)
{
    std::vector<PointIn> a(n ? n : 1), b(n ? n : 1);
    const size_t m1 = ktslice_weight_cull(in, n, weight_cull, a.data());
    if (m1 == 0) return 0;
    const size_t m2 = ktslice_voxel_grid(a.data(), m1, leaf, b.data(), n, 0, 0);
    std::vector<PointOut> o(m2 ? m2 : 1);
    ktslice_normals(b.data(), m2, k, leaf, o.data());
    const size_t m = std::min(m2, cap);
    memcpy(out48, o.data(), m * sizeof(PointOut));
    return m;
}

}
