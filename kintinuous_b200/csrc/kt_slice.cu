// kintinuous_b200 -- post-processing of an extracted cloud slice ON THE GPU, before it leaves the device.
//
// Replaces (reference, src/backend/CloudSliceProcessor.cpp:97-162, a CPU thread behind the tracker; SURVEY.md section 8 row f1):
//   weight cull (alpha >= -cw)                                               :104-121
//   pcl::VoxelGrid<PointXYZRGB>, leaf = voxel edge (one centroid per leaf)   :126-148     PCL 1.7.2 filters/impl/voxel_grid.hpp
//   pcl::NormalEstimation, KdTree, setKSearch(20), viewpoint (0,0,0)         :150-160     PCL 1.7.2 features/normal_3d.h, common/impl/{centroid,eigen}.hpp
//   pcl::concatenateFields -> PointXYZRGBNormal                              :162
// PCL is a third-party dependency that is not under the reference checkout; its published 1.7.2 algorithms are restated on the CPU by the test
// suite's checker (tests/test_slice_oracle.py pins it) and re-designed here:
//   * no sort, no kd-tree: the leaf grid itself is the spatial index.  A BIT PER LEAF (dx*dy*dz bits, 0.6 MB for a 17-plane slab of a
//     512^3 volume) marks occupied leaves; a prefix sum of the words' popcounts turns (word, bit) into the output slot, which is
//     PCL's output order (ascending leaf index) by construction;
//   * centroids accumulate in 64-bit fixed point (2^-32 m) with integer atomics: order-independent, hence deterministic run to run
//     (PCL's float sums depend on std::sort's unspecified order inside a leaf); colours are integer sums, divided as PCL divides them;
//   * the 20 nearest neighbours are found EXACTLY by one warp per point scanning the cube of +-r leaves around the point's leaf
//     (r = 3, 4, ...; a point outside the cube is farther than r leaves, so the search stops as soon as the 20th candidate is nearer),
//     candidates ranked by (squared distance, slot) -- the order the oracle uses -- in ONE pass (rank = number of smaller candidates);
//   * the 3x3 covariance is taken about the query point (PCL's single-pass float sum of raw coordinates loses ~3 digits to
//     cancellation for clouds metres away from the origin) and its smallest eigenpair comes from PCL's analytic eigen33 in FP64;
//     normal flipped towards the viewpoint (0,0,0), curvature = lambda0 / trace.
// Tolerances against the oracle (tests/test_gpu_slice.py): same leaves, same count; centroid <= 2e-6 m; colours exact; normals compared
// by angle (PCL's own cancellation noise is measured in the test against an FP64 recomputation).
// Bound: HBM-trivial (32 B in + 48 B out per point, a few MB per slice); the kNN pass is latency / issue bound.
#include "kt_ops.h"
#include "../../include/kintinuous_b200.h"

namespace kt {

namespace {

enum { SL_THREADS = 256, NRM_THREADS = 128, KNN_MAX = 32, CAND_CAP = 768, R_CAP = 10 };     // normals: 4 warps x 768 candidates x 8 B = 24 KB of shared memory

struct SliceGrid { int min_b[3]; int div_b[3]; float inv_leaf; float leaf; unsigned long long cells; };

__device__ __forceinline__ unsigned int ord_f(float f) { unsigned int u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__host__ __device__ __forceinline__ float unord_f(unsigned int u) { u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}

// bounds[0..2] = min (ordered uint), bounds[3..5] = max, bounds[6] = kept count
__global__ void __launch_bounds__(SL_THREADS)
slice_bounds_kernel(const kt_point_xyzrgb* __restrict__ in, unsigned int n, int weight_cull, unsigned int* __restrict__ bounds)
{
    unsigned int mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u}, cnt = 0;
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4 lo = __ldg(reinterpret_cast<const uint4*>(in) + (size_t)i * 2);
        const unsigned int rgba = __ldg(reinterpret_cast<const unsigned int*>(in) + (size_t)i * 8 + 4);
        if (weight_cull > 0 && (int)(rgba >> 24) < weight_cull) continue;
        const unsigned int ox = ord_f(__uint_as_float(lo.x)), oy = ord_f(__uint_as_float(lo.y)), oz = ord_f(__uint_as_float(lo.z));
        mn[0] = min(mn[0], ox); mn[1] = min(mn[1], oy); mn[2] = min(mn[2], oz);
        mx[0] = max(mx[0], ox); mx[1] = max(mx[1], oy); mx[2] = max(mx[2], oz);
        ++cnt;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o)); mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o)); }
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((threadIdx.x & 31) == 0 && cnt) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { atomicMin(&bounds[a], mn[a]); atomicMax(&bounds[3 + a], mx[a]); }
        atomicAdd(&bounds[6], cnt);
    }
}

// leaf of a point exactly as VoxelGrid::applyFilter computes it: static_cast<int>(floor(x * inverse_leaf) - static_cast<float>(min_b))
__device__ __forceinline__ bool leaf_of(const SliceGrid& g, float x, float y, float z, int& i0, int& i1, int& i2)
{
    i0 = (int)(floorf(__fmul_rn(x, g.inv_leaf)) - (float)g.min_b[0]);
    i1 = (int)(floorf(__fmul_rn(y, g.inv_leaf)) - (float)g.min_b[1]);
    i2 = (int)(floorf(__fmul_rn(z, g.inv_leaf)) - (float)g.min_b[2]);
    return (unsigned)i0 < (unsigned)g.div_b[0] && (unsigned)i1 < (unsigned)g.div_b[1] && (unsigned)i2 < (unsigned)g.div_b[2];
}
__device__ __forceinline__ unsigned long long leaf_index(const SliceGrid& g, int i0, int i1, int i2)
{ return ((unsigned long long)i2 * g.div_b[1] + i1) * g.div_b[0] + i0; }

__global__ void __launch_bounds__(SL_THREADS)
slice_mark_kernel(const kt_point_xyzrgb* __restrict__ in, unsigned int n, int weight_cull, const SliceGrid g, unsigned int* __restrict__ mask)
{
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4 lo = __ldg(reinterpret_cast<const uint4*>(in) + (size_t)i * 2);
        const unsigned int rgba = __ldg(reinterpret_cast<const unsigned int*>(in) + (size_t)i * 8 + 4);
        if (weight_cull > 0 && (int)(rgba >> 24) < weight_cull) continue;
        int i0, i1, i2;
        if (!leaf_of(g, __uint_as_float(lo.x), __uint_as_float(lo.y), __uint_as_float(lo.z), i0, i1, i2)) continue;
        const unsigned long long l = leaf_index(g, i0, i1, i2);
        atomicOr(&mask[l >> 5], 1u << (unsigned)(l & 31));
    }
}

// exclusive prefix sum of popc(mask[w]) in three passes: per-block totals, scan of the totals (one block), final offsets
enum { SCAN_ITEMS = 8, SCAN_BLOCK = SL_THREADS * SCAN_ITEMS };

__device__ __forceinline__ unsigned int block_exclusive_scan(unsigned int v, unsigned int* s_warp, unsigned int& total)
{
    const unsigned int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= (unsigned)o) inc += t; }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        unsigned int w = lane < SL_THREADS / 32 ? s_warp[lane] : 0u, winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned int t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= (unsigned)o) winc += t; }
        if (lane < SL_THREADS / 32) s_warp[lane] = winc - w;
        if (lane == 31) s_warp[32] = winc;
    }
    __syncthreads();
    total = s_warp[32];
    const unsigned int r = s_warp[wid] + inc - v;
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(SL_THREADS)
scan_block_totals_kernel(const unsigned int* __restrict__ mask, size_t words, unsigned int* __restrict__ block_tot)
{
    __shared__ unsigned int s_warp[33];
    const size_t base = (size_t)blockIdx.x * SCAN_BLOCK + (size_t)threadIdx.x * SCAN_ITEMS;
    unsigned int v = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) if (base + k < words) v += __popc(mask[base + k]);
    unsigned int total;
    block_exclusive_scan(v, s_warp, total);
    if (threadIdx.x == 0) block_tot[blockIdx.x] = total;
}

__global__ void __launch_bounds__(SL_THREADS)
scan_totals_kernel(unsigned int* __restrict__ block_tot, unsigned int nblocks, unsigned int* __restrict__ n_out)
{
    __shared__ unsigned int s_warp[33];
    unsigned int carry = 0;
    for (unsigned int b0 = 0; b0 < nblocks; b0 += SL_THREADS) {
        const unsigned int i = b0 + threadIdx.x;
        const unsigned int v = i < nblocks ? block_tot[i] : 0u;
        unsigned int total;
        const unsigned int ex = block_exclusive_scan(v, s_warp, total);
        if (i < nblocks) block_tot[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) *n_out = carry;
}

__global__ void __launch_bounds__(SL_THREADS)
scan_final_kernel(const unsigned int* __restrict__ mask, size_t words, const unsigned int* __restrict__ block_off, unsigned int* __restrict__ word_off)
{
    __shared__ unsigned int s_warp[33];
    const size_t base = (size_t)blockIdx.x * SCAN_BLOCK + (size_t)threadIdx.x * SCAN_ITEMS;
    unsigned int c[SCAN_ITEMS], v = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) { c[k] = base + k < words ? __popc(mask[base + k]) : 0; v += c[k]; }
    unsigned int total;
    unsigned int ex = block_exclusive_scan(v, s_warp, total) + block_off[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) { if (base + k < words) word_off[base + k] = ex; ex += c[k]; }
}

__device__ __forceinline__ unsigned int slot_of(const unsigned int* __restrict__ mask, const unsigned int* __restrict__ word_off, unsigned long long l)
{
    const unsigned int w = mask[l >> 5], b = (unsigned int)(l & 31);
    return word_off[l >> 5] + __popc(w & ((1u << b) - 1u));
}

struct SliceAcc { unsigned long long sx, sy, sz; unsigned int r, g, b, n; unsigned long long leaf; };     // 48 B per occupied leaf

__global__ void __launch_bounds__(SL_THREADS)
slice_accumulate_kernel(const kt_point_xyzrgb* __restrict__ in, unsigned int n, int weight_cull, const SliceGrid g,
                        const unsigned int* __restrict__ mask, const unsigned int* __restrict__ word_off, SliceAcc* __restrict__ acc)
{
    for (unsigned int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint4 lo = __ldg(reinterpret_cast<const uint4*>(in) + (size_t)i * 2);
        const unsigned int rgba = __ldg(reinterpret_cast<const unsigned int*>(in) + (size_t)i * 8 + 4);
        if (weight_cull > 0 && (int)(rgba >> 24) < weight_cull) continue;
        const float x = __uint_as_float(lo.x), y = __uint_as_float(lo.y), z = __uint_as_float(lo.z);
        int i0, i1, i2;
        if (!leaf_of(g, x, y, z, i0, i1, i2)) continue;
        const unsigned long long l = leaf_index(g, i0, i1, i2);
        SliceAcc* a = acc + slot_of(mask, word_off, l);
        // 2^-32 m fixed point, two's complement in an unsigned word: exact for |x| < 2^31 m, associative => deterministic
        atomicAdd(&a->sx, (unsigned long long)__double2ll_rn((double)x * 4294967296.0));
        atomicAdd(&a->sy, (unsigned long long)__double2ll_rn((double)y * 4294967296.0));
        atomicAdd(&a->sz, (unsigned long long)__double2ll_rn((double)z * 4294967296.0));
        atomicAdd(&a->r, (rgba >> 16) & 0xffu); atomicAdd(&a->g, (rgba >> 8) & 0xffu); atomicAdd(&a->b, rgba & 0xffu);
        if (atomicAdd(&a->n, 1u) == 0u) a->leaf = l;
    }
}

// centroid + colour of every occupied leaf -> the first 32 bytes of the 48-byte output point (normals are filled in by the kNN pass)
__global__ void __launch_bounds__(SL_THREADS)
slice_centroid_kernel(const SliceAcc* __restrict__ acc, unsigned int n_out, unsigned int cap, kt_point_xyzrgbnormal* __restrict__ out)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out || i >= cap) return;
    const SliceAcc a = acc[i];
    const double inv = 1.0 / ((double)a.n * 4294967296.0);
    kt_point_xyzrgbnormal p;
    p.x = (float)((double)(long long)a.sx * inv); p.y = (float)((double)(long long)a.sy * inv); p.z = (float)((double)(long long)a.sz * inv);
    p.data3 = 1.0f;
    const float cnt = (float)a.n;
    // VoxelGrid: centroid /= count in float, then (int) truncation of each channel; the alpha byte of the packed colour is 0
    p.r = (uint8_t)(int)__fdiv_rn((float)a.r, cnt); p.g = (uint8_t)(int)__fdiv_rn((float)a.g, cnt); p.b = (uint8_t)(int)__fdiv_rn((float)a.b, cnt); p.a = 0;
    p.nx = p.ny = p.nz = 0.f; p.data_n3 = 0.f; p.curvature = 0.f; p.pad[0] = p.pad[1] = 0.f;
    out[i] = p;
}

// ---- PCL 1.7.2 common/impl/eigen.hpp: computeRoots / computeRoots2 / eigen33 (smallest eigenpair), in FP64 ----
__device__ void compute_roots2(double b, double c, double* roots)
{
    roots[0] = 0.0;
    double d = b * b - 4.0 * c;
    if (d < 0.0) d = 0.0;
    const double sd = sqrt(d);
    roots[2] = 0.5 * (b + sd);
    roots[1] = 0.5 * (b - sd);
}
__device__ void compute_roots(const double* m, double* roots)
{
    const double c0 = m[0] * m[4] * m[8] + 2.0 * m[1] * m[2] * m[5] - m[0] * m[5] * m[5] - m[4] * m[2] * m[2] - m[8] * m[1] * m[1];
    const double c1 = m[0] * m[4] - m[1] * m[1] + m[0] * m[8] - m[2] * m[2] + m[4] * m[8] - m[5] * m[5];
    const double c2 = m[0] + m[4] + m[8];
    if (fabs(c0) < 2.220446049250313e-16) { compute_roots2(c2, c1, roots); return; }
    const double s_inv3 = 1.0 / 3.0, s_sqrt3 = 1.7320508075688772;
    const double c2_over_3 = c2 * s_inv3;
    double a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
    if (a_over_3 > 0.0) a_over_3 = 0.0;
    const double half_b = 0.5 * (c0 + c2_over_3 * (2.0 * c2_over_3 * c2_over_3 - c1));
    double q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
    if (q > 0.0) q = 0.0;
    const double rho = sqrt(-a_over_3);
    const double theta = atan2(sqrt(-q), half_b) * s_inv3;
    const double cos_theta = cos(theta), sin_theta = sin(theta);
    roots[0] = c2_over_3 + 2.0 * rho * cos_theta;
    roots[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
    roots[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
    double t;
    if (roots[0] >= roots[1]) { t = roots[0]; roots[0] = roots[1]; roots[1] = t; }
    if (roots[1] >= roots[2]) { t = roots[1]; roots[1] = roots[2]; roots[2] = t; if (roots[0] >= roots[1]) { t = roots[0]; roots[0] = roots[1]; roots[1] = t; } }
    if (roots[0] <= 0.0) compute_roots2(c2, c1, roots);
}
__device__ void eigen33_smallest(const double* mat, double* eigenvalue, double* vec)
{
    double scale = 0.0;
    for (int i = 0; i < 9; ++i) scale = fmax(scale, fabs(mat[i]));
    if (scale <= 2.2250738585072014e-308) scale = 1.0;
    double s[9];
    for (int i = 0; i < 9; ++i) s[i] = mat[i] / scale;
    double roots[3];
    compute_roots(s, roots);
    *eigenvalue = roots[0] * scale;
    s[0] -= roots[0]; s[4] -= roots[0]; s[8] -= roots[0];
    const double v1[3] = {s[1] * s[5] - s[2] * s[4], s[2] * s[3] - s[0] * s[5], s[0] * s[4] - s[1] * s[3]};
    const double v2[3] = {s[1] * s[8] - s[2] * s[7], s[2] * s[6] - s[0] * s[8], s[0] * s[7] - s[1] * s[6]};
    const double v3[3] = {s[4] * s[8] - s[5] * s[7], s[5] * s[6] - s[3] * s[8], s[3] * s[7] - s[4] * s[6]};
    const double l1 = v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2], l2 = v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2], l3 = v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2];
    const double* v; double l;
    if (l1 >= l2 && l1 >= l3) { v = v1; l = l1; } else if (l2 >= l1 && l2 >= l3) { v = v2; l = l2; } else { v = v3; l = l3; }
    const double inv = 1.0 / sqrt(l);
    vec[0] = v[0] * inv; vec[1] = v[1] * inv; vec[2] = v[2] * inv;
}

// One warp per point: exact k nearest neighbours through the leaf grid, covariance about the query point, smallest eigenvector.
__global__ void __launch_bounds__(NRM_THREADS)
slice_normals_kernel(kt_point_xyzrgbnormal* __restrict__ pts, const SliceAcc* __restrict__ acc, unsigned int n_out, int k, const SliceGrid g,
                     const unsigned int* __restrict__ mask, const unsigned int* __restrict__ word_off)
{
    // a candidate = ONE 64-bit key (bits of the squared distance, which is >= 0 so its bit pattern orders like its value) << 32 | slot:
    // (distance, slot) order is unsigned integer order, one shared-memory load and one compare per pair in the ranking pass
    __shared__ unsigned long long s_key[NRM_THREADS / 32][CAND_CAP];
    __shared__ float s_sd[NRM_THREADS / 32][KNN_MAX];
    __shared__ unsigned int s_si[NRM_THREADS / 32][KNN_MAX];
    const unsigned int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long* ck = s_key[wid]; float* sd = s_sd[wid]; unsigned int* si = s_si[wid];
    const int kk = min(k, (int)min(n_out, (unsigned int)KNN_MAX));
    for (unsigned int q = blockIdx.x * (NRM_THREADS / 32) + wid; q < n_out; q += gridDim.x * (NRM_THREADS / 32)) {
        const float qx = pts[q].x, qy = pts[q].y, qz = pts[q].z;
        const unsigned long long l = acc[q].leaf;
        const int c0 = (int)(l % g.div_b[0]), c1 = (int)((l / g.div_b[0]) % g.div_b[1]), c2 = (int)(l / ((unsigned long long)g.div_b[0] * g.div_b[1]));
        unsigned int ncand = 0;
        bool done = false;
        // r starts at 3: on a surface sampled at one point per leaf the 20th neighbour sits ~2.5 leaves away, so the +-2 cube almost never
        // passes the stop test and would only cost a second gather + ranking
        for (int r = 3; r <= R_CAP && !done; ++r) {
            const bool covers = c0 - r <= 0 && c1 - r <= 0 && c2 - r <= 0 && c0 + r >= g.div_b[0] - 1 && c1 + r >= g.div_b[1] - 1 && c2 + r >= g.div_b[2] - 1;
            unsigned int m = 0;
            const int side = 2 * r + 1, ncell = side * side * side;
            const float inv_side = 1.0f / (float)side;
            for (int cb = 0; cb < ncell; cb += 32) {
                const int c = cb + lane;
                bool hit = false; unsigned int slot = 0; float d = 0.f;
                if (c < ncell) {
                    // c = (cz * side + cy) * side + cx without integer division (exact: c < 2^14, side <= 21)
                    const int cq = __float2int_rz(((float)c + 0.5f) * inv_side), cz = __float2int_rz(((float)cq + 0.5f) * inv_side);
                    const int x = c0 - r + (c - cq * side), y = c1 - r + (cq - cz * side), z = c2 - r + cz;
                    if ((unsigned)x < (unsigned)g.div_b[0] && (unsigned)y < (unsigned)g.div_b[1] && (unsigned)z < (unsigned)g.div_b[2]) {
                        const unsigned long long ll = leaf_index(g, x, y, z);
                        const unsigned int w = mask[ll >> 5];
                        if ((w >> (unsigned)(ll & 31)) & 1u) {
                            slot = word_off[ll >> 5] + __popc(w & ((1u << (unsigned)(ll & 31)) - 1u));
                            const float dx = pts[slot].x - qx, dy = pts[slot].y - qy, dz = pts[slot].z - qz;
                            d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                            hit = true;
                        }
                    }
                }
                const unsigned int b = __ballot_sync(0xffffffffu, hit);
                const unsigned int pos = m + __popc(b & ((1u << lane) - 1u));
                if (hit && pos < CAND_CAP) ck[pos] = ((unsigned long long)__float_as_uint(d) << 32) | slot;
                m += __popc(b);
            }
            __syncwarp();
            if (m > CAND_CAP) break;                                   // cannot happen with one point per leaf before r = 5; the whole-cloud path below is exact anyway
            if ((int)m >= kk || covers) {
                // the kk smallest (distance, slot) pairs by RANK: a candidate's rank is the number of candidates before it in (distance, slot)
                // order (slots are unique, so ranks are); every lane ranks its candidates against all m (shared-memory broadcast reads) and
                // the ones with rank < kk drop into place -- one pass, no kk rounds of warp arg-min
                const int take = min(kk, (int)m);
                for (unsigned int j = lane; j < m; j += 32) {
                    const unsigned long long key = ck[j];
                    int rank = 0;
                    for (unsigned int i = 0; i < m; ++i) rank += ck[i] < key ? 1 : 0;
                    if (rank < take) { sd[rank] = __uint_as_float((unsigned int)(key >> 32)); si[rank] = (unsigned int)key; }
                }
                __syncwarp();
                const float dk = sd[take - 1];
                // a point outside the cube of +-r leaves is farther than r leaves from the query along some axis
                const float reach = ((float)r - 0.001f) * g.leaf;
                if (covers || ((int)m >= kk && dk <= reach * reach)) { done = true; ncand = (unsigned int)take; }
                __syncwarp();
            }
        }
        if (!done) {
            // isolated point (fewer than kk points within R_CAP leaves): successive minima of (distance, slot) over the whole cloud
            float ld = -1.f; unsigned int li = 0;
            for (int t = 0; t < kk; ++t) {
                float bd = 3.0e38f; unsigned int bi = 0xffffffffu;
                for (unsigned int sl = lane; sl < n_out; sl += 32) {
                    const float dx = pts[sl].x - qx, dy = pts[sl].y - qy, dz = pts[sl].z - qz;
                    const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                    const bool after = t == 0 || d > ld || (d == ld && sl > li);
                    if (after && (d < bd || (d == bd && sl < bi))) { bd = d; bi = sl; }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float od = __shfl_xor_sync(0xffffffffu, bd, o); const unsigned int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                    if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
                }
                if (lane == 0) { sd[t] = bd; si[t] = bi; }
                ld = bd; li = bi;
            }
            __syncwarp();
            ncand = (unsigned int)kk;
        }
        // covariance about the query point over the ncand selected neighbours (lanes 0 .. ncand-1), FP64
        double a[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        if (lane < ncand) {
            const unsigned int s = si[lane];
            const double dx = (double)pts[s].x - (double)qx, dy = (double)pts[s].y - (double)qy, dz = (double)pts[s].z - (double)qz;
            a[0] = dx * dx; a[1] = dx * dy; a[2] = dx * dz; a[3] = dy * dy; a[4] = dy * dz; a[5] = dz * dz; a[6] = dx; a[7] = dy; a[8] = dz;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int j = 0; j < 9; ++j) a[j] += __shfl_xor_sync(0xffffffffu, a[j], o);
        if (lane == 0) {
            float nx, ny, nz, curv;
            if (ncand < 3) { nx = ny = nz = curv = qnan(); }
            else {
                const double inv = 1.0 / (double)ncand;
                for (int j = 0; j < 9; ++j) a[j] *= inv;
                double cov[9];
                cov[0] = a[0] - a[6] * a[6]; cov[1] = a[1] - a[6] * a[7]; cov[2] = a[2] - a[6] * a[8];
                cov[4] = a[3] - a[7] * a[7]; cov[5] = a[4] - a[7] * a[8]; cov[8] = a[5] - a[8] * a[8];
                cov[3] = cov[1]; cov[6] = cov[2]; cov[7] = cov[5];
                double ev, v[3];
                eigen33_smallest(cov, &ev, v);
                const double tr = cov[0] + cov[4] + cov[8];
                curv = tr != 0.0 ? (float)fabs(ev / tr) : 0.f;
                // flipNormalTowardsViewpoint(point, 0, 0, 0): flip if (vp - p) . n < 0
                const double cs = -(double)qx * v[0] - (double)qy * v[1] - (double)qz * v[2];
                if (cs < 0) { v[0] = -v[0]; v[1] = -v[1]; v[2] = -v[2]; }
                nx = (float)v[0]; ny = (float)v[1]; nz = (float)v[2];
            }
            pts[q].nx = nx; pts[q].ny = ny; pts[q].nz = nz; pts[q].curvature = curv;
        }
        __syncwarp();
    }
}

int grid_for(size_t n) { size_t b = (n + SL_THREADS - 1) / SL_THREADS; const size_t cap = (size_t)device_info().sm_count * 8; return (int)(b < 1 ? 1 : (b > cap ? cap : b)); }

} // namespace

// Workspace of one slice: grown on demand, owned by the caller (tracker context or operator scratch).
int slice_ws_reserve(SliceWorkspace* ws, size_t words, size_t n_points)
{
    if (ws->words_cap < words) {
        if (ws->mask) cudaFree(ws->mask);
        if (ws->word_off) cudaFree(ws->word_off);
        if (ws->block_tot) cudaFree(ws->block_tot);
        ws->mask = 0; ws->word_off = 0; ws->block_tot = 0; ws->words_cap = 0;
        const size_t w = words + words / 4 + 1024;
        KT_CUDA(cudaMalloc((void**)&ws->mask, w * sizeof(unsigned int)));
        KT_CUDA(cudaMalloc((void**)&ws->word_off, w * sizeof(unsigned int)));
        KT_CUDA(cudaMalloc((void**)&ws->block_tot, ((w + SCAN_BLOCK - 1) / SCAN_BLOCK + 1) * sizeof(unsigned int)));
        ws->words_cap = w;
    }
    if (ws->acc_cap < n_points) {
        if (ws->acc) cudaFree(ws->acc);
        ws->acc = 0; ws->acc_cap = 0;
        const size_t m = n_points + n_points / 4 + 1024;
        KT_CUDA(cudaMalloc((void**)&ws->acc, m * sizeof(SliceAcc)));
        ws->acc_cap = m;
    }
    if (!ws->bounds) {
        KT_CUDA(cudaMalloc((void**)&ws->bounds, 8 * sizeof(unsigned int)));
        KT_CUDA(cudaMallocHost((void**)&ws->bounds_host, 8 * sizeof(unsigned int)));
    }
    return 0;
}

void slice_ws_free(SliceWorkspace* ws)
{
    if (ws->mask) cudaFree(ws->mask);
    if (ws->word_off) cudaFree(ws->word_off);
    if (ws->block_tot) cudaFree(ws->block_tot);
    if (ws->acc) cudaFree(ws->acc);
    if (ws->bounds) cudaFree(ws->bounds);
    if (ws->bounds_host) cudaFreeHost(ws->bounds_host);
    SliceWorkspace z = {0, 0, 0, 0, 0, 0, 0, 0};
    *ws = z;
}

// CloudSliceProcessor.cpp:97-162 on a device-resident slice.  Two host synchronisations (the leaf grid's extent and the output count
// decide allocation sizes); everything else is stream-ordered.  *count = processed points (capped at capacity).
int process_slice(const void* points_dev, size_t n, int weight_cull, float leaf, int k_search, void* out_dev, size_t capacity, size_t* count,
                  SliceWorkspace* ws, cudaStream_t s)
{
    if (count) *count = 0;
    if (n == 0) return 0;
    if (n > 0xfffffff0ull) { set_error("process_slice: more than 2^32 points"); return KT_ERR_INVALID; }
    if (!(leaf > 0.f) || k_search < 1 || k_search > KNN_MAX) { set_error("process_slice: leaf must be > 0 and 1 <= k <= %d", (int)KNN_MAX); return KT_ERR_INVALID; }
    int r = slice_ws_reserve(ws, 1, 1); if (r) return r;
    const kt_point_xyzrgb* in = (const kt_point_xyzrgb*)points_dev;
    const unsigned int init[8] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u, 0u};
    memcpy(ws->bounds_host, init, sizeof(init));
    KT_CUDA(cudaMemcpyAsync(ws->bounds, ws->bounds_host, sizeof(init), cudaMemcpyHostToDevice, s));
    slice_bounds_kernel<<<grid_for(n), SL_THREADS, 0, s>>>(in, (unsigned int)n, weight_cull, ws->bounds);
    KT_LAUNCH_CHECK();
    KT_CUDA(cudaMemcpyAsync(ws->bounds_host, ws->bounds, 8 * sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const unsigned int kept = ws->bounds_host[6];
    if (kept == 0) return 0;                                             // "after culling weights the cloud might be empty" (:124)
    SliceGrid g;
    g.leaf = leaf; g.inv_leaf = 1.0f / leaf;                             // inverse_leaf_size_ = 1 / leaf_size_ (float)
    float mn[3], mx[3];
    for (int a = 0; a < 3; ++a) { mn[a] = unord_f(ws->bounds_host[a]); mx[a] = unord_f(ws->bounds_host[3 + a]); }
    // voxel_grid.hpp: overflow check, then min_b / max_b / div_b
    const long long dx = (long long)((mx[0] - mn[0]) * g.inv_leaf) + 1, dy = (long long)((mx[1] - mn[1]) * g.inv_leaf) + 1, dz = (long long)((mx[2] - mn[2]) * g.inv_leaf) + 1;
    if (dx * dy * dz > 2147483647LL) {
        set_error("process_slice: the leaf grid has %lld x %lld x %lld cells, more than INT_MAX (pcl::VoxelGrid refuses it as well and returns the cloud unfiltered)", dx, dy, dz);
        return KT_ERR_INVALID;
    }
    for (int a = 0; a < 3; ++a) {
        g.min_b[a] = (int)floorf(mn[a] * g.inv_leaf);
        const int max_b = (int)floorf(mx[a] * g.inv_leaf);
        g.div_b[a] = max_b - g.min_b[a] + 1;
    }
    g.cells = (unsigned long long)g.div_b[0] * g.div_b[1] * g.div_b[2];
    const size_t words = (size_t)((g.cells + 31) / 32);
    if ((r = slice_ws_reserve(ws, words, kept))) return r;
    KT_CUDA(cudaMemsetAsync(ws->mask, 0, words * sizeof(unsigned int), s));
    slice_mark_kernel<<<grid_for(n), SL_THREADS, 0, s>>>(in, (unsigned int)n, weight_cull, g, ws->mask);
    KT_LAUNCH_CHECK();
    const unsigned int nblocks = (unsigned int)((words + SCAN_BLOCK - 1) / SCAN_BLOCK);
    scan_block_totals_kernel<<<nblocks, SL_THREADS, 0, s>>>(ws->mask, words, ws->block_tot);
    KT_LAUNCH_CHECK();
    scan_totals_kernel<<<1, SL_THREADS, 0, s>>>(ws->block_tot, nblocks, ws->bounds + 7);
    KT_LAUNCH_CHECK();
    scan_final_kernel<<<nblocks, SL_THREADS, 0, s>>>(ws->mask, words, ws->block_tot, ws->word_off);
    KT_LAUNCH_CHECK();
    KT_CUDA(cudaMemsetAsync(ws->acc, 0, (size_t)kept * sizeof(SliceAcc), s));
    slice_accumulate_kernel<<<grid_for(n), SL_THREADS, 0, s>>>(in, (unsigned int)n, weight_cull, g, ws->mask, ws->word_off, (SliceAcc*)ws->acc);
    KT_LAUNCH_CHECK();
    KT_CUDA(cudaMemcpyAsync(ws->bounds_host + 7, ws->bounds + 7, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const unsigned int n_out = ws->bounds_host[7];
    if ((size_t)n_out > capacity) { set_error("process_slice: %u processed points do not fit the output capacity %zu", n_out, capacity); return KT_ERR_CAPACITY; }
    kt_point_xyzrgbnormal* out = (kt_point_xyzrgbnormal*)out_dev;
    slice_centroid_kernel<<<div_up((int)n_out, SL_THREADS), SL_THREADS, 0, s>>>((const SliceAcc*)ws->acc, n_out, (unsigned int)capacity, out);
    KT_LAUNCH_CHECK();
    {
        const int warps_per_block = NRM_THREADS / 32;
        int blocks = div_up((int)n_out, warps_per_block);
        const int cap = device_info().sm_count * 16;
        if (blocks > cap) blocks = cap;
        slice_normals_kernel<<<blocks, NRM_THREADS, 0, s>>>(out, (const SliceAcc*)ws->acc, n_out, k_search, g, ws->mask, ws->word_off);
        KT_LAUNCH_CHECK();
    }
    if (count) *count = n_out;
    return 0;
}

} // namespace kt
