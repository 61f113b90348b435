// kintinuous_b200 -- weld keyed marching-cubes meshes into one: the mesh half of the map export (kt_get_map_mesh with weld).
//
// Stands in for (reference, src/backend/MeshGenerator.cpp:37-191, the `-nos` branch of MeshGenerator::save): there the whole map is
// voxel-gridded and triangulated again by PCL's greedy projection.  Here the slice meshes come from marching cubes over boxes of one
// cyclic TSDF (kt_mesh.cu), whose TSDF is gone after the shift, so nothing can be re-triangulated; what marching cubes gives instead is
// exact integer identity: every vertex lies on one edge of the global voxel lattice and every triangle belongs to one global cell.
// Meshes of overlapping boxes are therefore reconciled exactly, without a distance threshold (contract restated in numpy by the test
// suite's weld_oracle.weld):
//   * cell winner: a global cell keeps the triangles of the highest-numbered mesh that has triangles there (for the tracker the latest
//     slice, whose TSDF fused the most frames); every other mesh's triangles in that cell are dropped;
//   * vertex weld: only vertices a kept triangle uses are kept; of those on one global edge, the highest-numbered mesh's represents them
//     (within one mesh an edge occurs once); its 32 bytes are copied unchanged;
//   * order: vertices ascend by (gz, gy, gx, axis), triangles by cell and within a cell in the winning mesh's order -- kt_op_mesh_volume's
//     order, so welding the keyed meshes of overlapping boxes of one volume gives exactly the mesh of the union box.
// Design: one bounds pass (min / max of the lattice coordinates, and the input checks) -> 64-bit keys relative to the minimum, packed
// x fastest -> a stable CUB radix sort of (cell key, triangle) and, over the used vertices only, of (edge key, vertex): the inputs are
// concatenated in mesh order, so a stable sort orders equal keys by mesh -> head flags and scans pick the winners and the
// representatives -> triangle indices remapped by binary search in the unique edge keys (as kt_mesh.cu's find_vertex).  Atomics only
// in the bounds and the repeated-cell count, never in anything that decides the output order: two calls give byte-identical output.
// Scratch is allocated per call and freed before returning (the export runs between frames); a failed allocation returns KT_ERR_CUDA
// and leaves no CUDA error behind.  Three host synchronisations: the bounds, the used-vertex count, the output counts.
#include "kt_ops.h"
#include "../../include/kintinuous_b200.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>

namespace kt {

namespace {

enum { WELD_THREADS = 256 };

struct WeldGrid { int min[3]; unsigned long long ex, exy; };

__device__ __forceinline__ unsigned long long cell_key(const WeldGrid& g, int4 c)
{
    return (unsigned long long)(c.x - g.min[0]) + (unsigned long long)(c.y - g.min[1]) * g.ex + (unsigned long long)(c.z - g.min[2]) * g.exy;
}
__device__ __forceinline__ unsigned long long edge_key(const WeldGrid& g, int4 e) { return 3ull * cell_key(g, e) + (unsigned long long)e.w; }

__device__ __forceinline__ uint3 load_tri(const uint32_t* tris, unsigned long long t)
{ return make_uint3(__ldg(&tris[3 * t]), __ldg(&tris[3 * t + 1]), __ldg(&tris[3 * t + 2])); }

// the mesh element i belongs to: the last m with off[m] <= i (empty meshes are skipped)
__device__ __forceinline__ int mesh_of(const unsigned long long* off, int n_meshes, unsigned long long i)
{
    int lo = 0, hi = n_meshes;                          // first m with off[m] > i, minus one
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(&off[mid]) <= i) lo = mid + 1; else hi = mid; }
    return lo - 1;
}

// bounds[0..2] = min, [3..5] = max of gx, gy, gz over edges and cells; bounds[6] = bad records (axis outside 0..2, index outside its mesh)
__global__ void __launch_bounds__(WELD_THREADS)
weld_bounds_kernel(const int4* __restrict__ edges, unsigned long long nv, const int4* __restrict__ cells, const uint32_t* __restrict__ tris,
                   unsigned long long nt, const unsigned long long* __restrict__ voff, const unsigned long long* __restrict__ toff, int n_meshes,
                   int* __restrict__ bounds)
{
    int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {INT_MIN, INT_MIN, INT_MIN}, bad = 0;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nv + nt; i += stride) {
        int4 c;
        if (i < nv) {
            c = __ldg(&edges[i]);
            if ((unsigned)c.w > 2u) ++bad;
        } else {
            const unsigned long long t = i - nv;
            c = __ldg(&cells[t]);
            const int m = mesh_of(toff, n_meshes, t);
            const unsigned long long n = __ldg(&voff[m + 1]) - __ldg(&voff[m]);
            const uint3 v = load_tri(tris, t);
            if (v.x >= n || v.y >= n || v.z >= n) ++bad;
        }
        mn[0] = min(mn[0], c.x); mn[1] = min(mn[1], c.y); mn[2] = min(mn[2], c.z);
        mx[0] = max(mx[0], c.x); mx[1] = max(mx[1], c.y); mx[2] = max(mx[2], c.z);
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

__global__ void __launch_bounds__(WELD_THREADS)
weld_cell_keys_kernel(const int4* __restrict__ cells, unsigned int nt, const WeldGrid g, unsigned long long* __restrict__ keys, unsigned int* __restrict__ idx)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nt) { keys[i] = cell_key(g, __ldg(&cells[i])); idx[i] = i; }
}

// head[i] = 1 where a run of equal sorted keys starts
__global__ void __launch_bounds__(WELD_THREADS)
weld_heads_kernel(const unsigned long long* __restrict__ keys, unsigned int n, unsigned int* __restrict__ head)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}

// the winner of every cell: the mesh of its last sorted triangle (the sort is stable and the input in mesh order)
__global__ void __launch_bounds__(WELD_THREADS)
weld_winner_kernel(const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ idx, const unsigned int* __restrict__ seg, unsigned int n,
                   const unsigned long long* __restrict__ toff, int n_meshes, int* __restrict__ win)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (i == n - 1 || keys[i + 1] != keys[i])) win[seg[i] - 1] = mesh_of(toff, n_meshes, idx[i]);
}

// keep[i]: sorted triangle i belongs to its cell's winner; its vertices are then marked used.  counters[0] += cells with a loser.
__global__ void __launch_bounds__(WELD_THREADS)
weld_keep_kernel(const unsigned int* __restrict__ idx, const unsigned int* __restrict__ head, const unsigned int* __restrict__ seg, unsigned int n,
                 const int* __restrict__ win, const uint32_t* __restrict__ tris, const unsigned long long* __restrict__ voff,
                 const unsigned long long* __restrict__ toff, int n_meshes, unsigned int* __restrict__ keep, unsigned int* __restrict__ used,
                 unsigned long long* __restrict__ counters)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned int t = idx[i];
    const int m = mesh_of(toff, n_meshes, t);
    const bool k = m == win[seg[i] - 1];
    keep[i] = k ? 1u : 0u;
    if (head[i] && !k) atomicAdd(&counters[0], 1ull);            // the first triangle of the cell is not the winner's: repeated cell
    if (k) {
        const uint3 v = load_tri(tris, t);
        const unsigned long long b = __ldg(&voff[m]);
        used[b + v.x] = 1u; used[b + v.y] = 1u; used[b + v.z] = 1u;
    }
}

// the used vertices, compacted in input order, with their edge keys
__global__ void __launch_bounds__(WELD_THREADS)
weld_edge_keys_kernel(const int4* __restrict__ edges, const unsigned int* __restrict__ used, const unsigned int* __restrict__ slot, unsigned int nv,
                      const WeldGrid g, unsigned long long* __restrict__ keys, unsigned int* __restrict__ idx)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nv && used[i]) { keys[slot[i]] = edge_key(g, __ldg(&edges[i])); idx[slot[i]] = i; }
}

// tail[i] = 1 where a run of equal sorted keys ends: that vertex (the latest mesh's) represents the edge
__global__ void __launch_bounds__(WELD_THREADS)
weld_tails_kernel(const unsigned long long* __restrict__ keys, unsigned int n, unsigned int* __restrict__ tail)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) tail[i] = (i == n - 1 || keys[i + 1] != keys[i]) ? 1u : 0u;
}

__global__ void __launch_bounds__(WELD_THREADS)
weld_unique_kernel(const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ idx, const unsigned int* __restrict__ tail,
                   const unsigned int* __restrict__ uslot, unsigned int n, unsigned long long* __restrict__ ukeys, unsigned int* __restrict__ urep)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && tail[i]) { ukeys[uslot[i]] = keys[i]; urep[uslot[i]] = idx[i]; }
}

__global__ void __launch_bounds__(WELD_THREADS)
weld_write_verts_kernel(const uint4* __restrict__ verts, const unsigned int* __restrict__ urep, unsigned int nu, uint4* __restrict__ out)
{
    const unsigned int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < nu) { const unsigned int v = urep[j]; out[2 * j] = __ldg(&verts[2 * v]); out[2 * j + 1] = __ldg(&verts[2 * v + 1]); }
}

__device__ __forceinline__ unsigned int find_edge(const unsigned long long* keys, unsigned int n, unsigned long long key)
{
    unsigned int lo = 0, hi = n;                          // first index with keys[i] >= key; present by construction
    while (lo < hi) { const unsigned int mid = (lo + hi) >> 1; if (__ldg(&keys[mid]) < key) lo = mid + 1; else hi = mid; }
    return lo;
}

__global__ void __launch_bounds__(WELD_THREADS)
weld_write_tris_kernel(const unsigned int* __restrict__ idx, const unsigned int* __restrict__ keep, const unsigned int* __restrict__ tslot, unsigned int n,
                       const uint32_t* __restrict__ tris, const int4* __restrict__ edges, const unsigned long long* __restrict__ voff,
                       const unsigned long long* __restrict__ toff, int n_meshes, const WeldGrid g, const unsigned long long* __restrict__ ukeys,
                       unsigned int nu, uint32_t* __restrict__ out)
{
    const unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !keep[i]) return;
    const unsigned int t = idx[i];
    const unsigned long long b = __ldg(&voff[mesh_of(toff, n_meshes, t)]);
    const uint3 v = load_tri(tris, t);
    uint32_t* o = out + 3 * (size_t)tslot[i];
    o[0] = find_edge(ukeys, nu, edge_key(g, __ldg(&edges[b + v.x])));
    o[1] = find_edge(ukeys, nu, edge_key(g, __ldg(&edges[b + v.y])));
    o[2] = find_edge(ukeys, nu, edge_key(g, __ldg(&edges[b + v.z])));
}

int key_bits(unsigned long long kmax) { int b = 1; while (b < 64 && (kmax >> b) != 0) ++b; return b; }
unsigned int blocks_for(size_t n) { return (unsigned int)((n + WELD_THREADS - 1) / WELD_THREADS); }

} // namespace

int weld_meshes(const void* verts, const int32_t* vert_edges, const size_t* voff_h, const uint32_t* tris, const int32_t* tri_cells, const size_t* toff_h,
                int n_meshes, void* out_verts, size_t max_verts, uint32_t* out_tris, size_t max_tris, size_t* n_verts, size_t* n_tris,
                kt_weld_report* rep, cudaStream_t s)
{
    const char* who = "weld_meshes";
    *n_verts = 0; *n_tris = 0;
    kt_weld_report R; std::memset(&R, 0, sizeof(R));
    if (rep) *rep = R;
    if (n_meshes < 1 || !voff_h || !toff_h) { set_error("%s: at least one mesh and its offsets are needed", who); return KT_ERR_INVALID; }
    if (voff_h[0] != 0 || toff_h[0] != 0) { set_error("%s: the offsets must start at 0", who); return KT_ERR_INVALID; }
    for (int m = 0; m < n_meshes; ++m)
        if (voff_h[m + 1] < voff_h[m] || toff_h[m + 1] < toff_h[m]) { set_error("%s: the offsets of mesh %d descend", who, m); return KT_ERR_INVALID; }
    const size_t nv = voff_h[n_meshes], nt = toff_h[n_meshes];
    R.meshes = n_meshes; R.input_verts = nv; R.input_tris = nt;
    if (nv > 0x7fffffffull || nt > 0x7fffffffull) { set_error("%s: %zu vertices / %zu triangles, at most 2^31 - 1 each", who, nv, nt); return KT_ERR_INVALID; }
    if ((nv && (!verts || !vert_edges)) || (nt && (!tris || !tri_cells))) { set_error("%s: null input", who); return KT_ERR_INVALID; }
    if (nt == 0) { if (rep) *rep = R; return 0; }                  // nothing is meshed: nothing comes out
    if (nv == 0) { set_error("%s: triangles without vertices", who); return KT_ERR_INVALID; }

    Allocations mem(s);
    cudaEvent_t ev[4];
    for (int e = 0; e < 4; ++e) if (mem.event(&ev[e], cudaEventDefault, who)) return KT_ERR_CUDA;
    unsigned long long *voff = 0, *toff = 0, *counters = 0;
    int* bounds = 0;
    if (mem.device(&voff, (size_t)n_meshes + 1, who) || mem.device(&toff, (size_t)n_meshes + 1, who) || mem.device(&bounds, 8, who) ||
        mem.device(&counters, 2, who)) return KT_ERR_CUDA;
    std::vector<unsigned long long> vo(voff_h, voff_h + n_meshes + 1), to(toff_h, toff_h + n_meshes + 1);
    int host[8] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN, 0, 0};
    KT_CUDA(cudaEventRecord(ev[0], s));
    KT_CUDA(cudaMemcpyAsync(voff, vo.data(), vo.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(toff, to.data(), to.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(bounds, host, sizeof(host), cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemsetAsync(counters, 0, 2 * sizeof(unsigned long long), s));
    const int4* edges = (const int4*)vert_edges; const int4* cells = (const int4*)tri_cells; const uint32_t* tri3 = tris;
    {
        const size_t b = blocks_for(nv + nt), cap = (size_t)device_info().sm_count * 16;
        weld_bounds_kernel<<<(unsigned int)std::min(b, cap), WELD_THREADS, 0, s>>>(edges, nv, cells, tri3, nt, voff, toff, n_meshes, bounds);
        KT_LAUNCH_CHECK();
    }
    KT_CUDA(cudaMemcpyAsync(host, bounds, sizeof(host), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    if (host[6]) { set_error("%s: %d records have an axis outside 0..2 or a vertex index outside their mesh", who, host[6]); return KT_ERR_INVALID; }
    // packed keys: x fastest, relative to the minimum; the largest edge key is 3 ex ey ez - 1, checked against 2^62
    WeldGrid g;
    unsigned long long ext[3];
    for (int a = 0; a < 3; ++a) { g.min[a] = host[a]; ext[a] = (unsigned long long)((long long)host[3 + a] - (long long)host[a] + 1); }
    const unsigned long long LIM = 1ull << 62;
    if (ext[1] > LIM / ext[0] || ext[2] > LIM / (ext[0] * ext[1]) || ext[0] * ext[1] * ext[2] > LIM / 3) {
        set_error("%s: the keys span %llu x %llu x %llu voxels, beyond 2^62 edge keys", who, ext[0], ext[1], ext[2]); return KT_ERR_INVALID;
    }
    g.ex = ext[0]; g.exy = ext[0] * ext[1];
    const unsigned long long ncell = g.exy * ext[2];
    const int cbits = key_bits(ncell - 1), ebits = key_bits(3 * ncell - 1);
    const unsigned int NT = (unsigned int)nt, NV = (unsigned int)nv;

    // triangles: (cell key, index) sorted, winners, kept flags and their slots
    unsigned long long *tk0, *tk1; unsigned int *ti0, *ti1, *thead, *tseg, *tkeep, *tslot, *used, *vslot; int* win; unsigned char* tmp;
    if (mem.device(&tk0, nt, who) || mem.device(&tk1, nt, who) || mem.device(&ti0, nt, who) || mem.device(&ti1, nt, who) ||
        mem.device(&thead, nt, who) || mem.device(&tseg, nt, who) || mem.device(&tkeep, nt, who) || mem.device(&tslot, nt, who) ||
        mem.device(&win, nt, who) || mem.device(&used, nv, who) || mem.device(&vslot, nv, who)) return KT_ERR_CUDA;
    cub::DoubleBuffer<unsigned long long> tkb(tk0, tk1); cub::DoubleBuffer<unsigned int> tib(ti0, ti1);
    size_t sort_t = 0, sort_v = 0, scan_t = 0, scan_v = 0;
    KT_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_t, tkb, tib, NT, 0, cbits, s));
    KT_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_v, tkb, tib, NV, 0, ebits, s));
    KT_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_t, thead, tseg, NT, s));
    KT_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_v, used, vslot, NV, s));
    const size_t tmp_bytes = std::max(std::max(sort_t, sort_v), std::max(scan_t, scan_v));
    if (mem.device(&tmp, tmp_bytes, who)) return KT_ERR_CUDA;
    KT_CUDA(cudaMemsetAsync(used, 0, nv * sizeof(unsigned int), s));
    KT_CUDA(cudaEventRecord(ev[1], s));
    weld_cell_keys_kernel<<<blocks_for(nt), WELD_THREADS, 0, s>>>(cells, NT, g, tk0, ti0);
    KT_LAUNCH_CHECK();
    size_t have = tmp_bytes;
    KT_CUDA(cub::DeviceRadixSort::SortPairs(tmp, have, tkb, tib, NT, 0, cbits, s));
    const unsigned long long* tkey = tkb.Current(); const unsigned int* tidx = tib.Current();
    weld_heads_kernel<<<blocks_for(nt), WELD_THREADS, 0, s>>>(tkey, NT, thead);
    KT_LAUNCH_CHECK();
    have = tmp_bytes;
    KT_CUDA(cub::DeviceScan::InclusiveSum(tmp, have, thead, tseg, NT, s));         // 1-based cell number of every sorted triangle
    weld_winner_kernel<<<blocks_for(nt), WELD_THREADS, 0, s>>>(tkey, tidx, tseg, NT, toff, n_meshes, win);
    KT_LAUNCH_CHECK();
    weld_keep_kernel<<<blocks_for(nt), WELD_THREADS, 0, s>>>(tidx, thead, tseg, NT, win, tri3, voff, toff, n_meshes, tkeep, used, counters);
    KT_LAUNCH_CHECK();
    have = tmp_bytes;
    KT_CUDA(cub::DeviceScan::ExclusiveSum(tmp, have, tkeep, tslot, NT, s));
    have = tmp_bytes;
    KT_CUDA(cub::DeviceScan::ExclusiveSum(tmp, have, used, vslot, NV, s));
    unsigned int last[4];
    KT_CUDA(cudaMemcpyAsync(&last[0], tslot + NT - 1, 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(&last[1], tkeep + NT - 1, 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(&last[2], vslot + NV - 1, 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(&last[3], used + NV - 1, 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const unsigned int kept = last[0] + last[1], nused = last[2] + last[3];

    // used vertices: (edge key, index) sorted, one representative per edge
    unsigned long long *vk0, *vk1, *ukeys; unsigned int *vi0, *vi1, *vtail, *uslot, *urep;
    if (mem.device(&vk0, nused, who) || mem.device(&vk1, nused, who) || mem.device(&vi0, nused, who) || mem.device(&vi1, nused, who) ||
        mem.device(&vtail, nused, who) || mem.device(&uslot, nused, who) || mem.device(&ukeys, nused, who) || mem.device(&urep, nused, who)) return KT_ERR_CUDA;
    weld_edge_keys_kernel<<<blocks_for(nv), WELD_THREADS, 0, s>>>(edges, used, vslot, NV, g, vk0, vi0);
    KT_LAUNCH_CHECK();
    cub::DoubleBuffer<unsigned long long> vkb(vk0, vk1); cub::DoubleBuffer<unsigned int> vib(vi0, vi1);
    have = tmp_bytes;
    KT_CUDA(cub::DeviceRadixSort::SortPairs(tmp, have, vkb, vib, nused, 0, ebits, s));
    KT_CUDA(cudaEventRecord(ev[2], s));
    const unsigned long long* vkey = vkb.Current(); const unsigned int* vidx = vib.Current();
    weld_tails_kernel<<<blocks_for(nused), WELD_THREADS, 0, s>>>(vkey, nused, vtail);
    KT_LAUNCH_CHECK();
    have = tmp_bytes;
    KT_CUDA(cub::DeviceScan::ExclusiveSum(tmp, have, vtail, uslot, nused, s));
    weld_unique_kernel<<<blocks_for(nused), WELD_THREADS, 0, s>>>(vkey, vidx, vtail, uslot, nused, ukeys, urep);
    KT_LAUNCH_CHECK();
    unsigned long long cnt[2];
    KT_CUDA(cudaMemcpyAsync(&last[0], uslot + nused - 1, 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(&last[1], vtail + nused - 1, 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(cnt, counters, sizeof(cnt), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const unsigned int nu = last[0] + last[1];
    R.output_verts = nu; R.output_tris = kept; R.repeated_cells = cnt[0];
    R.dropped_triangles = nt - kept; R.merged_vertices = nused - nu;
    *n_verts = nu; *n_tris = kept;
    if (nu > max_verts || kept > max_tris || (nu && !out_verts) || (kept && !out_tris)) {
        if (rep) *rep = R;
        set_error("%s: %u vertices / %u triangles exceed the capacities", who, nu, kept); return KT_ERR_CAPACITY;
    }
    weld_write_verts_kernel<<<blocks_for(nu), WELD_THREADS, 0, s>>>((const uint4*)verts, urep, nu, (uint4*)out_verts);
    KT_LAUNCH_CHECK();
    weld_write_tris_kernel<<<blocks_for(nt), WELD_THREADS, 0, s>>>(tidx, tkeep, tslot, NT, tri3, edges, voff, toff, n_meshes, g, ukeys, nu, out_tris);
    KT_LAUNCH_CHECK();
    KT_CUDA(cudaEventRecord(ev[3], s));
    KT_CUDA(cudaStreamSynchronize(s));
    KT_CUDA(cudaEventElapsedTime(&R.sort_ms, ev[1], ev[2]));
    KT_CUDA(cudaEventElapsedTime(&R.weld_ms, ev[2], ev[3]));
    KT_CUDA(cudaEventElapsedTime(&R.total_ms, ev[0], ev[3]));
    if (rep) *rep = R;
    return 0;
}

} // namespace kt
