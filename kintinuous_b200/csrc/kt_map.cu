// kintinuous_b200 -- pcl::VoxelGrid over a whole map on the GPU: the overlap filter of the map export (kt_get_map_cloud with dedupe).
//
// Replaces (reference, src/backend/CloudSliceProcessor.cpp:180-231, `-nos`): one pcl::VoxelGrid<PointXYZRGBNormal> at the voxel edge over
// every slice's processed cloud, concatenated.  PCL 1.7.2 filters/impl/voxel_grid.hpp, applyFilter with downsample_all_data = true,
// min_points_per_voxel = 0, no filter field, is_dense = true, restated for both point types (kt_point_xyzrgb, kt_point_xyzrgbnormal):
//   * bounds: exact min / max of x, y, z (ordered-integer atomics); a non-finite x / y / z is refused;
//   * leaf of a point: i_k = (floor(p_k * inv) - (float)min_b_k), inv = 1.0f / leaf on the host, the product rounded (__fmul_rn, no
//     contraction), exactly as PCL writes it, but the leaf index i0 + i1 div0 + i2 div0 div1 is formed in 64 bits.  Where PCL's int
//     index does not overflow, the two are equal, so ascending keys are PCL's output order;
//   * a stable CUB radix sort of (key, point index) over only the key bits the grid needs: points of one leaf stay in input order (the
//     order the test suite's oracle fixes where PCL's std::sort leaves it unspecified);
//   * leaf starts by a head flag + exclusive scan; then one thread per leaf walks its points in sorted order with PCL's float
//     arithmetic: the accumulator starts at the first point (NdCopyPointEigenFunctor, so a -0.0 survives), every field (x, y, z; for
//     the 48-byte type also normal_x/y/z and curvature) and r, g, b (as floats) is added with __fadd_rn, divided by the count with
//     __fdiv_rn (the build's --prec-div=false would make '/' approximate), colour packed as (int)r << 16 | (int)g << 8 | (int)b
//     (alpha 0), data[3] = 1, data_n[3] = 0.  A NaN normal propagates as in PCL.
// The output is therefore bit-identical to the test suite's float32 restatement (map_oracle.py) except where a sum or a quotient is subnormal
// (the build flushes subnormals: --ftz=true) and in NaN payloads (the GPU returns the canonical NaN).
// Deliberate divergence: where PCL's int64 check dx * dy * dz > INT_MAX fires, PCL warns and returns the cloud UNFILTERED; this filter
// goes on with its 64-bit keys and reports *pcl_would_skip = 1.  Keys beyond 2^62 or min_b / max_b outside int: KT_ERR_INVALID.
// Workspace: allocated per call and freed before returning (the export runs between frames); a failed allocation returns KT_ERR_CUDA
// and leaves no CUDA error behind.  Two host synchronisations: the bounds (grid size) and the leaf count.
#include "kt_ops.h"
#include "../../include/kintinuous_b200.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cmath>
#include <cstring>

namespace kt {

namespace {

enum { MAP_THREADS = 256 };

__device__ __forceinline__ unsigned int ord_f(float f) { unsigned int u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
float unord_f(unsigned int u) { u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u; float f; memcpy(&f, &u, 4); return f; }

// x, y, z of record i (both point types start with x, y, z, data[3]; 16-byte aligned)
template <int REC> __device__ __forceinline__ float4 xyz_of(const unsigned char* __restrict__ in, size_t i)
{ return __ldg(reinterpret_cast<const float4*>(in + i * REC)); }

// bounds[0..2] = min (ordered uint), [3..5] = max, [6] = points with a non-finite x / y / z
template <int REC>
__global__ void __launch_bounds__(MAP_THREADS)
map_bounds_kernel(const unsigned char* __restrict__ in, size_t n, unsigned int* __restrict__ bounds)
{
    unsigned int mn[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, mx[3] = {0u, 0u, 0u}, bad = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4 p = xyz_of<REC>(in, i);
        if (!isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z)) { ++bad; continue; }
        const unsigned int o[3] = {ord_f(p.x), ord_f(p.y), ord_f(p.z)};
#pragma unroll
        for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], o[a]); mx[a] = max(mx[a], o[a]); }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o)); mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o)); }
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { atomicMin(&bounds[a], mn[a]); atomicMax(&bounds[3 + a], mx[a]); }
        if (bad) atomicAdd(&bounds[6], bad);
    }
}

struct MapGrid { float inv; float min_b[3]; unsigned long long mul1, mul2; };

template <int REC>
__global__ void __launch_bounds__(MAP_THREADS)
map_keys_kernel(const unsigned char* __restrict__ in, size_t n, const MapGrid g, unsigned long long* __restrict__ keys, unsigned int* __restrict__ idx)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4 p = xyz_of<REC>(in, i);
        // PCL: static_cast<int> (floor (p * inverse_leaf_size) - static_cast<float> (min_b)); every value here is >= 0 and < 2^33
        const unsigned long long i0 = (unsigned long long)(floorf(__fmul_rn(p.x, g.inv)) - g.min_b[0]);
        const unsigned long long i1 = (unsigned long long)(floorf(__fmul_rn(p.y, g.inv)) - g.min_b[1]);
        const unsigned long long i2 = (unsigned long long)(floorf(__fmul_rn(p.z, g.inv)) - g.min_b[2]);
        keys[i] = i0 + i1 * g.mul1 + i2 * g.mul2;
        idx[i] = (unsigned int)i;
    }
}

// head[i] = 1 where a leaf starts in the sorted keys
__global__ void __launch_bounds__(MAP_THREADS)
map_heads_kernel(const unsigned long long* __restrict__ keys, unsigned int n, unsigned int* __restrict__ head)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}

// starts[leaf] = first sorted position of the leaf; starts[leaves] = n, and *n_leaves
__global__ void __launch_bounds__(MAP_THREADS)
map_starts_kernel(const unsigned int* __restrict__ head, const unsigned int* __restrict__ slot, unsigned int n, unsigned int* __restrict__ starts,
                  unsigned int* __restrict__ n_leaves)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (head[i]) starts[slot[i]] = i;
    if (i == n - 1) { const unsigned int m = slot[i] + head[i]; starts[m] = n; *n_leaves = m; }
}

// the averaged fields of record p: x y z [nx ny nz curvature] r g b
template <int REC, int NF> __device__ __forceinline__ void map_fields(const unsigned char* __restrict__ p, float (&f)[NF])
{
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    f[0] = a.x; f[1] = a.y; f[2] = a.z;
    unsigned int rgba;
    if (REC == 48) {
        const float4 nrm = __ldg(reinterpret_cast<const float4*>(p + 16));
        const float2 cc = __ldg(reinterpret_cast<const float2*>(p + 32));
        f[3] = nrm.x; f[4] = nrm.y; f[5] = nrm.z; f[NF - 4] = cc.y;
        rgba = __float_as_uint(cc.x);
    } else {
        rgba = __ldg(reinterpret_cast<const unsigned int*>(p + 16));
    }
    f[NF - 3] = (float)((rgba >> 16) & 0xffu); f[NF - 2] = (float)((rgba >> 8) & 0xffu); f[NF - 1] = (float)(rgba & 0xffu);
}

// one thread per leaf: PCL's float centroid of its points in sorted order (see the file header)
template <int REC>
__global__ void __launch_bounds__(MAP_THREADS, 4)        // without the minimum ptxas caps the <48> instance at 32 registers and spills
map_centroid_kernel(const unsigned char* __restrict__ in, const unsigned int* __restrict__ idx, const unsigned int* __restrict__ starts,
                    unsigned int n_out, unsigned char* __restrict__ out)
{
    constexpr int NF = REC == 48 ? 10 : 6;
    const unsigned int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_out) return;
    const unsigned int b = starts[j], e = starts[j + 1];
    float acc[NF];
    map_fields<REC>(in + (size_t)__ldg(idx + b) * REC, acc);
    for (unsigned int k = b + 1; k < e; ++k) {
        float f[NF];
        map_fields<REC>(in + (size_t)__ldg(idx + k) * REC, f);
#pragma unroll
        for (int q = 0; q < NF; ++q) acc[q] = __fadd_rn(acc[q], f[q]);
    }
    const float cnt = __uint2float_rn(e - b);
#pragma unroll
    for (int q = 0; q < NF; ++q) acc[q] = __fdiv_rn(acc[q], cnt);
    const int rgb = (int)acc[NF - 3] << 16 | (int)acc[NF - 2] << 8 | (int)acc[NF - 1];
    unsigned char* o = out + (size_t)j * REC;
    reinterpret_cast<float4*>(o)[0] = make_float4(acc[0], acc[1], acc[2], 1.0f);
    if (REC == 48) {
        reinterpret_cast<float4*>(o)[1] = make_float4(acc[3], acc[4], acc[5], 0.0f);
        reinterpret_cast<float4*>(o)[2] = make_float4(__int_as_float(rgb), acc[6], 0.0f, 0.0f);
    } else {
        reinterpret_cast<float4*>(o)[1] = make_float4(__int_as_float(rgb), 0.0f, 0.0f, 0.0f);
    }
}

// x' = R x + t, n' = R n (kt_point_xyzrgbnormal records, in place), FP32 without contraction
__global__ void __launch_bounds__(MAP_THREADS)
map_rigid_kernel(kt_point_xyzrgbnormal* __restrict__ p, size_t n, const RigidF C)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float4 a = reinterpret_cast<float4*>(p + i)[0], b = reinterpret_cast<float4*>(p + i)[1];
        const float* R = C.R;
        const float x = a.x, y = a.y, z = a.z, nx = b.x, ny = b.y, nz = b.z;
        a.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[0], x), __fmul_rn(R[1], y)), __fmul_rn(R[2], z)), C.t[0]);
        a.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[3], x), __fmul_rn(R[4], y)), __fmul_rn(R[5], z)), C.t[1]);
        a.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[6], x), __fmul_rn(R[7], y)), __fmul_rn(R[8], z)), C.t[2]);
        b.x = __fadd_rn(__fadd_rn(__fmul_rn(R[0], nx), __fmul_rn(R[1], ny)), __fmul_rn(R[2], nz));
        b.y = __fadd_rn(__fadd_rn(__fmul_rn(R[3], nx), __fmul_rn(R[4], ny)), __fmul_rn(R[5], nz));
        b.z = __fadd_rn(__fadd_rn(__fmul_rn(R[6], nx), __fmul_rn(R[7], ny)), __fmul_rn(R[8], nz));
        reinterpret_cast<float4*>(p + i)[0] = a; reinterpret_cast<float4*>(p + i)[1] = b;
    }
}

// the same for kt_mesh_vertex records (x y z nx | ny nz rgba pad)
__global__ void __launch_bounds__(MAP_THREADS)
map_rigid_mesh_kernel(kt_mesh_vertex* __restrict__ p, size_t n, const RigidF C)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float4 a = reinterpret_cast<float4*>(p + i)[0], b = reinterpret_cast<float4*>(p + i)[1];
        const float* R = C.R;
        const float x = a.x, y = a.y, z = a.z, nx = a.w, ny = b.x, nz = b.y;
        a.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[0], x), __fmul_rn(R[1], y)), __fmul_rn(R[2], z)), C.t[0]);
        a.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[3], x), __fmul_rn(R[4], y)), __fmul_rn(R[5], z)), C.t[1]);
        a.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[6], x), __fmul_rn(R[7], y)), __fmul_rn(R[8], z)), C.t[2]);
        a.w = __fadd_rn(__fadd_rn(__fmul_rn(R[0], nx), __fmul_rn(R[1], ny)), __fmul_rn(R[2], nz));
        b.x = __fadd_rn(__fadd_rn(__fmul_rn(R[3], nx), __fmul_rn(R[4], ny)), __fmul_rn(R[5], nz));
        b.y = __fadd_rn(__fadd_rn(__fmul_rn(R[6], nx), __fmul_rn(R[7], ny)), __fmul_rn(R[8], nz));
        reinterpret_cast<float4*>(p + i)[0] = a; reinterpret_cast<float4*>(p + i)[1] = b;
    }
}

int grid_for(size_t n) { const size_t b = (n + MAP_THREADS - 1) / MAP_THREADS, cap = (size_t)device_info().sm_count * 16; return (int)(b < 1 ? 1 : (b > cap ? cap : b)); }

// Stage timing of one voxel_grid call (CUDA events on its stream)
struct MapEvents {
    cudaEvent_t e[4]; bool on;
    explicit MapEvents(bool want) : on(false) {
        for (int i = 0; i < 4; ++i) e[i] = 0;
        if (!want) return;
        on = true;
        for (int i = 0; i < 4; ++i) if (cudaEventCreate(&e[i]) != cudaSuccess) { cudaGetLastError(); on = false; }
    }
    ~MapEvents() { for (int i = 0; i < 4; ++i) if (e[i]) cudaEventDestroy(e[i]); }
    void mark(int i, cudaStream_t s) { if (on) cudaEventRecord(e[i], s); }
    float ms(int a, int b) { float t = 0.f; if (on && cudaEventElapsedTime(&t, e[a], e[b]) != cudaSuccess) { cudaGetLastError(); t = 0.f; } return t; }
};

template <int REC>
int voxel_grid_impl(const unsigned char* in, size_t n, float leaf, unsigned char* out, size_t capacity, size_t* count, int* pcl_would_skip,
                    float* ms2, cudaStream_t s)
{
    const char* who = "voxel_grid";
    MapEvents ev(ms2 != 0);
    Allocations mem(s);
    unsigned int host[7] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u};
    unsigned int* bounds = 0; unsigned char* w = 0; unsigned char* tmp = 0;
    int r = mem.device(&bounds, 7, "voxel_grid bounds"); if (r) return r;
    KT_CUDA(cudaMemcpyAsync(bounds, host, sizeof(host), cudaMemcpyHostToDevice, s));
    map_bounds_kernel<REC><<<grid_for(n), MAP_THREADS, 0, s>>>(in, n, bounds);
    KT_LAUNCH_CHECK();
    KT_CUDA(cudaMemcpyAsync(host, bounds, sizeof(host), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    if (host[6]) { set_error("%s: %u points have a non-finite x, y or z", who, host[6]); return KT_ERR_INVALID; }
    float mn[3], mx[3];
    for (int a = 0; a < 3; ++a) { mn[a] = unord_f(host[a]); mx[a] = unord_f(host[3 + a]); }
    MapGrid g; g.inv = 1.0f / leaf;                                   // inverse_leaf_size_ = 1 / leaf_size_ (float)
    long long min_b[3], div_b[3], top[3];
    for (int a = 0; a < 3; ++a) {
        const float lo = std::floor(mn[a] * g.inv), hi = std::floor(mx[a] * g.inv);
        if (!(lo >= -2147483648.0f && hi < 2147483648.0f)) {
            set_error("%s: the leaf grid's bounds (%g .. %g leaves on axis %d) do not fit an int", who, (double)lo, (double)hi, a); return KT_ERR_INVALID; }
        min_b[a] = (long long)lo; div_b[a] = (long long)hi - min_b[a] + 1;
        g.min_b[a] = lo;
        // largest leaf coordinate: floor(p * inv) - (float)min_b is a float difference, exact below 2^24, rounded above
        top[a] = (long long)(float)(div_b[a] - 1);
    }
    // largest key, checked against 2^62 (every product below stays under 2^64: each factor < 2^33, checked step by step)
    const unsigned long long LIM = 1ull << 62;
    const unsigned long long d0 = (unsigned long long)div_b[0], d1 = (unsigned long long)div_b[1];
    if (d1 > LIM / d0) { set_error("%s: the leaf grid has more than 2^62 cells", who); return KT_ERR_INVALID; }
    g.mul1 = d0; g.mul2 = d0 * d1;
    if ((unsigned long long)top[2] > LIM / g.mul2) { set_error("%s: the leaf grid has more than 2^62 cells", who); return KT_ERR_INVALID; }
    const unsigned long long kmax = (unsigned long long)top[0] + (unsigned long long)top[1] * g.mul1 + (unsigned long long)top[2] * g.mul2;
    if (kmax > LIM) { set_error("%s: the leaf grid has more than 2^62 cells", who); return KT_ERR_INVALID; }
    // voxel_grid.hpp's overflow check, in int64 as PCL computes it: PCL would return the cloud unfiltered
    const long long dx = (long long)((mx[0] - mn[0]) * g.inv) + 1, dy = (long long)((mx[1] - mn[1]) * g.inv) + 1, dz = (long long)((mx[2] - mn[2]) * g.inv) + 1;
    *pcl_would_skip = (__int128)dx * dy * dz > (__int128)2147483647 ? 1 : 0;
    int bits = 1;
    while (bits < 64 && (kmax >> bits) != 0) ++bits;

    // workspace: keys x 2, indices x 2, head flags, scan, starts (n + 1), leaf count
    const unsigned int nn = (unsigned int)n;
    const size_t off_k1 = (size_t)n * 8, off_i0 = off_k1 + (size_t)n * 8, off_i1 = off_i0 + (size_t)n * 4, off_h = off_i1 + (size_t)n * 4,
                 off_s = off_h + (size_t)n * 4, off_st = off_s + (size_t)n * 4, off_m = off_st + ((size_t)n + 1) * 4, total = off_m + 16;
    if ((r = mem.device(&w, total, "voxel_grid keys and indices"))) return r;
    unsigned long long* k0 = (unsigned long long*)w; unsigned long long* k1 = (unsigned long long*)(w + off_k1);
    unsigned int* i0 = (unsigned int*)(w + off_i0); unsigned int* i1 = (unsigned int*)(w + off_i1);
    unsigned int* head = (unsigned int*)(w + off_h); unsigned int* slot = (unsigned int*)(w + off_s);
    unsigned int* starts = (unsigned int*)(w + off_st); unsigned int* n_leaves = (unsigned int*)(w + off_m);
    cub::DoubleBuffer<unsigned long long> kb(k0, k1); cub::DoubleBuffer<unsigned int> vb(i0, i1);
    size_t sort_bytes = 0, scan_bytes = 0;
    KT_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, kb, vb, nn, 0, bits, s));
    KT_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, head, slot, nn, s));
    if ((r = mem.device(&tmp, std::max(sort_bytes, scan_bytes), "voxel_grid sort storage"))) return r;

    ev.mark(0, s);
    map_keys_kernel<REC><<<grid_for(n), MAP_THREADS, 0, s>>>(in, n, g, k0, i0);
    KT_LAUNCH_CHECK();
    KT_CUDA(cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, kb, vb, nn, 0, bits, s));
    ev.mark(1, s);
    const unsigned long long* keys = kb.Current(); const unsigned int* idx = vb.Current();
    const int blocks = (int)((n + MAP_THREADS - 1) / MAP_THREADS);
    map_heads_kernel<<<blocks, MAP_THREADS, 0, s>>>(keys, nn, head);
    KT_LAUNCH_CHECK();
    KT_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, head, slot, nn, s));
    map_starts_kernel<<<blocks, MAP_THREADS, 0, s>>>(head, slot, nn, starts, n_leaves);
    KT_LAUNCH_CHECK();
    unsigned int m = 0;
    KT_CUDA(cudaMemcpyAsync(&m, n_leaves, sizeof(m), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const unsigned int n_out = (unsigned int)std::min((size_t)m, capacity);
    if (out && n_out) {
        map_centroid_kernel<REC><<<div_up((int)n_out, MAP_THREADS), MAP_THREADS, 0, s>>>(in, idx, starts, n_out, out);
        KT_LAUNCH_CHECK();
    }
    ev.mark(2, s);
    KT_CUDA(cudaStreamSynchronize(s));
    if (ms2) { ms2[0] = ev.ms(0, 1); ms2[1] = ev.ms(1, 2); }
    *count = m;
    return 0;
}

} // namespace

int voxel_grid(const void* points_dev, size_t n, int kind, float leaf, void* out_dev, size_t capacity, size_t* count, int* pcl_would_skip,
               float* ms2, cudaStream_t s)
{
    *count = 0; *pcl_would_skip = 0;
    if (ms2) ms2[0] = ms2[1] = 0.f;
    if ((kind != 0 && kind != 1) || !(leaf > 0.f) || !std::isfinite(leaf) || (n && !points_dev)) { set_error("voxel_grid: kind must be 0 or 1, leaf > 0 and finite"); return KT_ERR_INVALID; }
    if (n > 0x7fffffffull) { set_error("voxel_grid: %zu points, at most 2^31 - 1", n); return KT_ERR_INVALID; }
    if (n == 0) return 0;
    return kind == 0 ? voxel_grid_impl<32>((const unsigned char*)points_dev, n, leaf, (unsigned char*)out_dev, capacity, count, pcl_would_skip, ms2, s)
                     : voxel_grid_impl<48>((const unsigned char*)points_dev, n, leaf, (unsigned char*)out_dev, capacity, count, pcl_would_skip, ms2, s);
}

int rigid_move(void* points_dev, size_t n, const RigidF& C, cudaStream_t s)
{
    if (!n) return 0;
    map_rigid_kernel<<<grid_for(n), MAP_THREADS, 0, s>>>((kt_point_xyzrgbnormal*)points_dev, n, C);
    KT_LAUNCH_CHECK();
    return 0;
}

int rigid_move_mesh(void* verts_dev, size_t n, const RigidF& C, cudaStream_t s)
{
    if (!n) return 0;
    map_rigid_mesh_kernel<<<grid_for(n), MAP_THREADS, 0, s>>>((kt_mesh_vertex*)verts_dev, n, C);
    KT_LAUNCH_CHECK();
    return 0;
}

} // namespace kt
