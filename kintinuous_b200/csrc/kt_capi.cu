// kintinuous_b200 -- operator-level C ABI (kt_op_*): one entry point per free function of the reference's
// src/frontend/cuda/internal.h:299-536, same argument meaning, synchronous semantics (results visible on return),
// status codes instead of exit(0).  The tracker-level ABI (kt_create / kt_process_frame / ...) is in kt_tracker.cu.
#include "kt_ops.h"
#include "kt_solve.cuh"
#include "kt_pgo.hpp"
#include "../../include/kintinuous_b200.h"
#include <cstring>
#include <cstddef>
#include <mutex>
#include <vector>
#include <algorithm>

using namespace kt;

namespace {

Intr intr4(const float* k) { Intr r = {k[0], k[1], k[2], k[3]}; return r; }
Mat33 mat33(const float* m) { Mat33 r; r.r0 = make_float3(m[0], m[1], m[2]); r.r1 = make_float3(m[3], m[4], m[5]); r.r2 = make_float3(m[6], m[7], m[8]); return r; }
cudaStream_t st(void* s) { return (cudaStream_t)s; }

// Scratch of the stateless operator calls (the reference keeps sumDataSE3 / outDataSE3 in its odometry objects and is not thread-safe
// either: internal.h:299-536 has static state in computeDerivativeImages and __device__ globals in extract.cu).  One set PER DEVICE
// (the device current at the call), and the calls that use it are serialised by a process-wide mutex, so operator calls from several
// host threads / on several devices are safe, just not concurrent.
struct OpScratch { Allocations mem; OdomState* state; float* partials; int* ipartials; unsigned int* counter; OdomState* host_state;
                   DeviceBuffer<float> ztable; SliceWorkspace slice_ws; MeshWorkspace mesh_ws; DeviceBuffer<unsigned long long> mesh_cells; SurfWorkspace surf_ws; PnpWorkspace pnp_ws;
                   SliceWorkspace fit_ws; DeviceBuffer<int> place_ints; };   // place_ints: kt_op_surf / kt_op_match_ratio counts in, counts out
enum { KT_MAX_DEVICES = 64 };
// Allocated once per device and never destroyed: no CUDA call may run in the static destructors at process exit.
OpScratch* g_ops_dev[KT_MAX_DEVICES];
std::mutex g_ops_mu;
OpScratch& ops_scratch()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= KT_MAX_DEVICES) dev = 0;
    if (!g_ops_dev[dev]) g_ops_dev[dev] = new OpScratch();
    return *g_ops_dev[dev];
}
#define g_ops (ops_scratch())
#define KT_OPS_LOCK() std::lock_guard<std::mutex> _ops_lock(g_ops_mu)

int ensure_scratch()
{
    if (g_ops.host_state) return 0;
    Allocations m; const char* W = "operator scratch";
    OdomState* state; float* partials; int* ipartials; unsigned int* counter; OdomState* host_state;
    int r;
    if ((r = m.device(&state, 1, W)) || (r = m.device(&partials, (size_t)MAX_PARTIALS * 32, W)) || (r = m.device(&ipartials, (size_t)MAX_PARTIALS * 2, W)) ||
        (r = m.device(&counter, 1, W)) || (r = m.pinned(&host_state, 1, W))) return r;
    KT_CUDA(cudaMemset(state, 0, sizeof(OdomState)));
    OpScratch& o = g_ops;
    o.mem = std::move(m); o.state = state; o.partials = partials; o.ipartials = ipartials; o.counter = counter; o.host_state = host_state;
    return 0;
}
// The volume operators' one requirement on vol (include/kintinuous_b200.h): a positive multiple of 8.  The y / z clear stores 16-byte
// words along a row and init_volume fills whole 16-byte words, so any other side would misalign those stores or leave voxels unwritten.
int check_vol(const char* who, int vol)
{
    if (vol <= 0 || vol % 8 != 0) { set_error("%s: vol %d is not a positive multiple of 8", who, vol); return KT_ERR_INVALID; }
    return KT_OK;
}

int ensure_ztable(int vol)
{
    const size_t n = vol > 0 ? (size_t)2 * vol : 0;
    return g_ops.ztable.grow(n, n, "operator z table");
}

} // namespace

extern "C" {

int kt_op_bilateral(const uint16_t* src, uint16_t* dst, int rows, int cols, void* s)
{ int r = bilateral(src, dst, rows, cols, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }

int kt_op_pyrdown(const uint16_t* src, uint16_t* dst, int sr, int sc, void* s)
{ int r = pyrdown(src, dst, sr, sc, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }

int kt_op_create_vmap(const float* k, const uint16_t* depth, float* vmap, int rows, int cols, void* s)
{ int r = create_vmap(intr4(k), depth, vmap, rows, cols, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }

int kt_op_create_nmap(const float* vmap, float* nmap, int rows, int cols, void* s)
{ int r = create_nmap(vmap, nmap, rows, cols, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }

int kt_op_create_maps(const float* k, const uint16_t* depth, float* vmap, float* nmap, int rows, int cols, void* s)
{
    MapsLevel L; L.depth = depth; L.vmap = vmap; L.nmap = nmap; L.rows = rows; L.cols = cols; L.k = intr4(k); L.vstale = 0; L.nstale = 0;
    int r = create_maps_pyramid(&L, 1, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK;
}

// the product's fused front end (bilateral_scale_kernel + frontend_pyramid_kernel) on caller buffers: what the tracker runs per frame
int kt_op_frontend(const uint16_t* depth_raw, const uint8_t* rgb, int rows, int cols, const float* k, int angle_color,
                   uint16_t* const* depths4, float* const* vmaps4, float* const* nmaps4, float* depth_scaled, float* cw, float* rgbf,
                   float* const* depth_m4, uint8_t* const* intensity4, int16_t* const* dIdx4, int16_t* const* dIdy4, void* s)
{
    if (!depth_raw || !rgb || !depths4 || !vmaps4 || !nmaps4) { set_error("kt_op_frontend: null argument"); return KT_ERR_INVALID; }
    int r = bilateral_scale(depth_raw, depths4[0], depth_scaled, rows, cols, intr4(k), angle_color != 0, st(s)); if (r) return r;
    FrontendArgs fa;
    fa.depth_f = depths4[0]; fa.depth_raw = depth_raw; fa.rgb = rgb; fa.rows = rows; fa.cols = cols; fa.k = intr4(k);
    fa.depths = depths4; fa.vmaps = vmaps4; fa.nmaps = nmaps4; fa.vstale = 0; fa.nstale = 0;
    fa.cw = cw; fa.rgbf = (float4*)rgbf; fa.angle_color = angle_color != 0; fa.cut_off = 6000;
    fa.depth_m = depth_m4; fa.intensity = intensity4; fa.dIdx = dIdx4; fa.dIdy = dIdy4;
    r = frontend_pyramid(fa, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_transform_maps(const float* vs, const float* ns, const float* R, const float* t, float* vd, float* nd, int rows, int cols, void* s)
{ int r = transform_maps(vs, ns, mat33(R), make_float3(t[0], t[1], t[2]), vd, nd, rows, cols, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }

int kt_op_resize_vmap(const float* in, float* out, int in_rows, int in_cols, void* s)
{ int r = resize_map(in, out, in_rows, in_cols, false, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }

int kt_op_resize_nmap(const float* in, float* out, int in_rows, int in_cols, void* s)
{ int r = resize_map(in, out, in_rows, in_cols, true, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }

int kt_op_icp_step(const float* Rcurr, const float* tcurr, const float* vmap_curr, const float* nmap_curr,
                   const float* Rprev_inv, const float* tprev, const float* k,
                   const float* vmap_g_prev, const float* nmap_g_prev, int rows, int cols,
                   float dist_thres, float angle_thres, float* A_host, float* b_host, float* residual_host, void* s)
{
    KT_OPS_LOCK();
    int r = ensure_scratch(); if (r) return r;
    OdomState* h = g_ops.host_state;
    std::memset(h, 0, sizeof(OdomState));
    std::memcpy(h->Rcurr, Rcurr, 36); std::memcpy(h->tcurr, tcurr, 12); std::memcpy(h->Rprev_inv, Rprev_inv, 36); std::memcpy(h->tprev, tprev, 12);
    KT_CUDA(cudaMemcpyAsync(g_ops.state, h, sizeof(OdomState), cudaMemcpyHostToDevice, st(s)));
    IcpLevelArgs a = {vmap_curr, nmap_curr, vmap_g_prev, nmap_g_prev, rows, cols, intr4(k), dist_thres, angle_thres};
    r = icp_iteration(a, g_ops.state, g_ops.partials, 0, 0, st(s)); if (r) return r;
    KT_CUDA(cudaMemcpyAsync(h->sums_icp, (char*)g_ops.state + offsetof(OdomState, sums_icp), 32 * sizeof(float), cudaMemcpyDeviceToHost, st(s)));
    KT_CUDA(cudaStreamSynchronize(st(s)));
    unpack_normal_equations(h->sums_icp, A_host, b_host);
    residual_host[0] = h->sums_icp[27]; residual_host[1] = h->sums_icp[28];
    return KT_OK;
}

int kt_op_integrate(const uint16_t* depth_raw, int rows, int cols, const float* k, const float* vs,
                    const float* Rinv, const float* t, float trunc, int16_t* tsdf, uint8_t* color, int vol,
                    const int* wrap, const uint8_t* rgb, const float* nmap_curr, int angle_color, float* depth_scaled, void* s)
{
    int r = check_vol("kt_op_integrate", vol); if (r) return r;
    KT_OPS_LOCK();
    r = ensure_ztable(vol); if (r) return r;
    r = scale_depth(depth_raw, depth_scaled, rows, cols, intr4(k), angle_color != 0, st(s)); if (r) return r;
    IntegrateArgs a; a.cw = 0; a.rgbf = 0; a.reset_words = 0; a.reset_count = 0; a.reset_stride = 1;
    a.depth_scaled = depth_scaled; a.rows = rows; a.cols = cols; a.k = intr4(k); a.volume_size = make_float3(vs[0], vs[1], vs[2]);
    a.Rinv = mat33(Rinv); a.t = make_float3(t[0], t[1], t[2]); a.trunc = trunc; a.tsdf = tsdf; a.color = color; a.vol = vol;
    a.wrap = make_int3(wrap[0], wrap[1], wrap[2]); a.rgb = rgb; a.nmap_curr = nmap_curr; a.angle_color = angle_color != 0;
    a.multi = 0; a.vv = single_volume(tsdf, color, vol);
    r = integrate(a, g_ops.ztable.get(), st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_raycast(const float* k, const float* R, const float* t, float trunc, const float* vs,
                  const int16_t* tsdf, int vol, float* vmap, float* nmap, int rows, int cols,
                  const int* wrap, uint8_t* vmap_color, const uint8_t* color, void* s)
{
    // a cell size the ray cast cannot divide by is wrong whatever the side, so it is named first (a side <= 0 has no cell: check_vol)
    if (vol > 0) { if (int r = check_cell_size(make_float3(vs[0], vs[1], vs[2]), vol)) return r; }
    if (int r = check_vol("kt_op_raycast", vol)) return r;
    RaycastArgs a = {};          // multi = 0 (one volume) and no field left for raycast() to read uninitialised
    a.k = intr4(k); a.R = mat33(R); a.t = make_float3(t[0], t[1], t[2]); a.trunc = trunc; a.volume_size = make_float3(vs[0], vs[1], vs[2]);
    a.tsdf = tsdf; a.color = color; a.vol = vol; a.wrap = make_int3(wrap[0], wrap[1], wrap[2]);
    for (int l = 0; l < LEVELS; ++l) { a.vmap[l] = vmap; a.nmap[l] = nmap; }
    a.rows = rows; a.cols = cols; a.vmap_color = vmap_color; a.n_levels = 1;
    int r = raycast(a, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_extract_slice(const int16_t* tsdf, const float* vs, int vol, kt_point_xyzrgb* out, size_t capacity,
                        const int* wrap, const uint8_t* color, int minX, int maxX, int minY, int maxY, int minZ, int maxZ,
                        int subsample, const int* real_wrap, size_t* count, void* s)
{
    int r = check_vol("kt_op_extract_slice", vol); if (r) return r;
    KT_OPS_LOCK();
    r = ensure_scratch(); if (r) return r;
    KT_CUDA(cudaMemsetAsync(g_ops.counter, 0, sizeof(unsigned int), st(s)));
    r = extract_slice(tsdf, make_float3(vs[0], vs[1], vs[2]), vol, out, capacity, make_int3(wrap[0], wrap[1], wrap[2]), color,
                      minX, maxX, minY, maxY, minZ, maxZ, subsample, make_int3(real_wrap[0], real_wrap[1], real_wrap[2]), g_ops.counter, st(s));
    if (r) return r;
    unsigned int n = 0;
    KT_CUDA(cudaMemcpyAsync(&n, g_ops.counter, sizeof(n), cudaMemcpyDeviceToHost, st(s)));
    KT_CUDA(cudaStreamSynchronize(st(s)));
    if (count) *count = n < capacity ? n : capacity;
    return KT_OK;
}

int kt_op_process_slice(const kt_point_xyzrgb* points_dev, size_t n, int weight_cull, float leaf, int k_search, kt_point_xyzrgbnormal* out_dev, size_t capacity,
                        size_t* count, void* s)
{
    KT_OPS_LOCK();
    return process_slice(points_dev, n, weight_cull, leaf, k_search, out_dev, capacity, count, &g_ops.slice_ws, st(s));
}

int kt_op_voxel_grid(const void* points_dev, size_t n, int kind, float leaf, void* out_dev, size_t capacity, size_t* count, int* pcl_would_skip, void* s)
{
    if (!count || !pcl_would_skip || (capacity && !out_dev)) { set_error("kt_op_voxel_grid: bad argument"); return KT_ERR_INVALID; }
    return voxel_grid(points_dev, n, kind, leaf, out_dev, capacity, count, pcl_would_skip, 0, st(s));
}

int kt_op_mesh_volume(const int16_t* tsdf, const uint8_t* color, int vol, const float* vs, const int* wrap, const int* real_wrap,
                      int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int weight_cull, kt_mesh_vertex* verts, size_t max_verts,
                      uint32_t* tris, size_t max_tris, size_t* n_verts, size_t* n_tris, void* s)
{
    if (int r = check_vol("kt_op_mesh_volume", vol)) return r;
    if (!tsdf || !color || !vs || !wrap || !real_wrap || !n_verts || !n_tris) { set_error("kt_op_mesh_volume: bad argument"); return KT_ERR_INVALID; }
    if (minX < 0 || minY < 0 || minZ < 0 || maxX > vol || maxY > vol || maxZ > vol) { set_error("kt_op_mesh_volume: box outside [0, vol]"); return KT_ERR_INVALID; }
    KT_OPS_LOCK();
    MeshArgs a;
    a.tsdf = tsdf; a.color = color; a.vol = vol; a.volume_size = make_float3(vs[0], vs[1], vs[2]);
    a.wrap = make_int3(wrap[0], wrap[1], wrap[2]); a.real_wrap = make_int3(real_wrap[0], real_wrap[1], real_wrap[2]);
    a.minX = minX; a.maxX = maxX; a.minY = minY; a.maxY = maxY; a.minZ = minZ; a.maxZ = maxZ; a.weight_cull = weight_cull;
    size_t nv = 0, nt = 0;
    int r = mesh_count(a, &g_ops.mesh_ws, &nv, &nt, st(s)); if (r) return r;
    *n_verts = nv; *n_tris = nt;
    if (nv > max_verts || nt > max_tris) { set_error("kt_op_mesh_volume: %zu vertices / %zu triangles exceed the capacities", nv, nt); return KT_ERR_CAPACITY; }
    r = mesh_emit(a, &g_ops.mesh_ws, nv, verts, tris, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_mesh_volume_keyed(const int16_t* tsdf, const uint8_t* color, int vol, const float* vs, const int* wrap, const int* real_wrap,
                            int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int weight_cull, kt_mesh_vertex* verts, int32_t* vert_edges,
                            size_t max_verts, uint32_t* tris, int32_t* tri_cells, size_t max_tris, size_t* n_verts, size_t* n_tris, void* s)
{
    if (int r = check_vol("kt_op_mesh_volume_keyed", vol)) return r;
    if (!tsdf || !color || !vs || !wrap || !real_wrap || !n_verts || !n_tris) { set_error("kt_op_mesh_volume_keyed: bad argument"); return KT_ERR_INVALID; }
    if (minX < 0 || minY < 0 || minZ < 0 || maxX > vol || maxY > vol || maxZ > vol) { set_error("kt_op_mesh_volume_keyed: box outside [0, vol]"); return KT_ERR_INVALID; }
    KT_OPS_LOCK();
    MeshArgs a;
    a.tsdf = tsdf; a.color = color; a.vol = vol; a.volume_size = make_float3(vs[0], vs[1], vs[2]);
    a.wrap = make_int3(wrap[0], wrap[1], wrap[2]); a.real_wrap = make_int3(real_wrap[0], real_wrap[1], real_wrap[2]);
    a.minX = minX; a.maxX = maxX; a.minY = minY; a.maxY = maxY; a.minZ = minZ; a.maxZ = maxZ; a.weight_cull = weight_cull;
    size_t nv = 0, nt = 0;
    int r = mesh_count(a, &g_ops.mesh_ws, &nv, &nt, st(s)); if (r) return r;
    *n_verts = nv; *n_tris = nt;
    if (nv > max_verts || nt > max_tris || (nv && (!verts || !vert_edges)) || (nt && (!tris || !tri_cells))) {
        set_error("kt_op_mesh_volume_keyed: %zu vertices / %zu triangles exceed the capacities", nv, nt); return KT_ERR_CAPACITY;
    }
    if ((r = g_ops.mesh_cells.grow(nt, nt, "operator mesh cells"))) return r;
    r = mesh_emit(a, &g_ops.mesh_ws, nv, verts, tris, st(s), nullptr, g_ops.mesh_cells.get()); if (r) return r;
    if ((r = mesh_global_keys(a, g_ops.mesh_ws.keys.get(), nv, true, vert_edges, st(s)))) return r;
    if ((r = mesh_global_keys(a, g_ops.mesh_cells.get(), nt, false, tri_cells, st(s)))) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_mesh_bricks(const uint64_t* keys, const int16_t* tsdf, const uint8_t* color, size_t n_bricks, const float* vs, int vol, int weight_cull,
                      kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris, size_t* n_verts, size_t* n_tris, void* s)
{
    const char* who = "kt_op_mesh_bricks";
    if (!vs || !n_verts || !n_tris || (n_bricks && (!keys || !tsdf || !color))) { set_error("%s: bad argument", who); return KT_ERR_INVALID; }
    if (vol <= 0) { set_error("%s: vol %d is not positive", who, vol); return KT_ERR_INVALID; }
    const MeshOutput out = [&](size_t nv, size_t nt, void** v, uint32_t** t) -> int {
        if (!verts && !tris) return 1;
        if (nv > max_verts || nt > max_tris || !verts || (nt && !tris)) {
            set_error("%s: %zu vertices / %zu triangles exceed the capacities", who, nv, nt); return KT_ERR_CAPACITY; }
        *v = verts; *t = tris;
        return 0;
    };
    BrickSet set = {(const unsigned long long*)keys, tsdf, color, n_bricks};
    return mesh_bricks(set, make_float3(vs[0], vs[1], vs[2]), vol, weight_cull, out, n_verts, n_tris, nullptr, st(s));
}

int kt_op_weld_meshes(const kt_mesh_vertex* verts, const int32_t* vert_edges, const size_t* vert_offsets, const uint32_t* tris, const int32_t* tri_cells,
                      const size_t* tri_offsets, int n_meshes, kt_mesh_vertex* out_verts, size_t max_verts, uint32_t* out_tris, size_t max_tris,
                      size_t* n_verts, size_t* n_tris, kt_weld_report* report, void* s)
{
    if (!n_verts || !n_tris) { set_error("kt_op_weld_meshes: bad argument"); return KT_ERR_INVALID; }
    return weld_meshes(verts, vert_edges, vert_offsets, tris, tri_cells, tri_offsets, n_meshes, out_verts, max_verts, out_tris, max_tris, n_verts, n_tris,
                       report, st(s));
}

int kt_op_deform_weights(const float* node_pos, const uint64_t* node_times, int n_nodes, const void* pts, int kind, const uint64_t* times,
                         size_t n, int32_t* ids, double* weights, void* s)
{
    if (!node_pos || !node_times || (n && (!pts || !times || !ids || !weights))) { set_error("kt_op_deform_weights: bad argument"); return KT_ERR_INVALID; }
    int r = deform_weights(node_pos, node_times, n_nodes, pts, kind, times, n, ids, weights, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_deform_optimise(const float* node_pos, int n_nodes, const float* con_src, const double* con_dst, const int32_t* con_ids,
                          const double* con_w, size_t m, double* params, kt_deform_report* report, void* s)
{
    if (!node_pos || !params || !report || n_nodes < 0 || (m && (!con_src || !con_dst || !con_ids || !con_w))) {
        set_error("kt_op_deform_optimise: bad argument"); return KT_ERR_INVALID;
    }
    std::vector<float> pos((size_t)n_nodes * 3), src(m * 3); std::vector<double> dst(m * 3), w(m * 4); std::vector<int32_t> ids(m * 4);
    KT_CUDA(cudaMemcpyAsync(pos.data(), node_pos, pos.size() * sizeof(float), cudaMemcpyDeviceToHost, st(s)));
    if (m) {
        KT_CUDA(cudaMemcpyAsync(src.data(), con_src, src.size() * sizeof(float), cudaMemcpyDeviceToHost, st(s)));
        KT_CUDA(cudaMemcpyAsync(dst.data(), con_dst, dst.size() * sizeof(double), cudaMemcpyDeviceToHost, st(s)));
        KT_CUDA(cudaMemcpyAsync(ids.data(), con_ids, ids.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st(s)));
        KT_CUDA(cudaMemcpyAsync(w.data(), con_w, w.size() * sizeof(double), cudaMemcpyDeviceToHost, st(s)));
    }
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return deform_optimise(pos.data(), n_nodes, src.data(), dst.data(), ids.data(), w.data(), m, params, report, st(s));
}

// isam::Slam::batch_optimization (iSAMInterface.cpp:136-140) over a caller's graph
int kt_op_pgo_optimise(const double* poses, int n_nodes, const kt_pgo_factor* factors, int n_factors, double* out, kt_pgo_report* report, void* s)
{
    static_assert(sizeof(kt_pgo_factor) == sizeof(PgoFactor) && offsetof(kt_pgo_factor, z) == offsetof(PgoFactor, z), "kt_pgo_factor layout");
    if (!poses || !factors || !out || !report || n_nodes < 2 || n_factors < n_nodes) { set_error("kt_op_pgo_optimise: bad argument"); return KT_ERR_INVALID; }
    std::vector<PgoFactor> f(n_factors);
    KT_CUDA(cudaMemcpyAsync(f.data(), factors, f.size() * sizeof(PgoFactor), cudaMemcpyDeviceToHost, st(s)));
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return pgo_optimise(poses, n_nodes, f.data(), n_factors, out, report, st(s));
}

int kt_op_deform_apply(const float* node_pos, const double* params, int n_nodes, const int32_t* ids, const double* weights, const void* in,
                       void* out, int kind, size_t n, void* s)
{
    if (!node_pos || !params || n_nodes <= 0 || (n && (!ids || !weights || !in || !out))) { set_error("kt_op_deform_apply: bad argument"); return KT_ERR_INVALID; }
    int r = deform_apply(node_pos, params, n_nodes, ids, weights, in, out, kind, n, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_clear_volume(int axis, int back, int16_t* tsdf, uint8_t* color, int vol, int current, int delta, void* s)
{
    int r = check_vol("kt_op_clear_volume", vol); if (r) return r;
    r = clear_volume(axis, back, tsdf, color, vol, current, delta, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK;
}

int kt_op_init_volume(int16_t* tsdf, uint8_t* color, int vol, void* s)
{
    int r = check_vol("kt_op_init_volume", vol); if (r) return r;
    r = init_volume(tsdf, color, vol, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK;
}

int kt_op_short_depth_to_metres(const uint16_t* src, float* dst, int rows, int cols, int cut, void* s)
{ int r = short_depth_to_metres(src, dst, rows, cols, cut, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }
int kt_op_pyrdown_gauss_f(const float* src, float* dst, int sr, int sc, void* s)
{ int r = pyrdown_gauss_f(src, dst, sr, sc, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }
int kt_op_bgr_to_intensity(const uint8_t* rgb, uint8_t* dst, int rows, int cols, void* s)
{ int r = bgr_to_intensity(rgb, dst, rows, cols, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }
int kt_op_pyrdown_uchar_gauss(const uint8_t* src, uint8_t* dst, int sr, int sc, void* s)
{ int r = pyrdown_uchar_gauss(src, dst, sr, sc, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }
int kt_op_derivative_images(const uint8_t* src, int16_t* dx, int16_t* dy, int rows, int cols, void* s)
{ int r = derivative_images(src, dx, dy, rows, cols, st(s)); if (r) return r; KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK; }
int kt_op_project_to_point_cloud(const float* depth, float* cloud, int rows, int cols, const double* k, int level, void* s)
{
    const int div = 1 << level;                                    // IntrDoublePrecision::operator() (internal.h:268-272)
    int r = project_to_point_cloud(depth, cloud, rows, cols, k[0] / div, k[1] / div, k[2] / div, k[3] / div, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK;
}

int kt_op_rgb_residual(float min_scale, const int16_t* dIdx, const int16_t* dIdy, const float* last_depth, const float* next_depth,
                       const uint8_t* last_image, const uint8_t* next_image, void* corres, int rows, int cols,
                       float max_depth_delta, const float* kt3, const float* krkinv9, int* sigma_sum, int* count, void* s)
{
    KT_OPS_LOCK();
    int r = ensure_scratch(); if (r) return r;
    OdomState* h = g_ops.host_state;
    std::memset(h, 0, sizeof(OdomState));
    std::memcpy(h->krkinv, krkinv9, 36); std::memcpy(h->kt, kt3, 12);
    KT_CUDA(cudaMemcpyAsync(g_ops.state, h, sizeof(OdomState), cudaMemcpyHostToDevice, st(s)));
    RgbLevelArgs a; std::memset(&a, 0, sizeof(a));
    a.dIdx = dIdx; a.dIdy = dIdy; a.last_depth = last_depth; a.next_depth = next_depth; a.last_image = last_image; a.next_image = next_image;
    a.corres = corres; a.rows = rows; a.cols = cols; a.min_scale = min_scale; a.max_depth_delta = max_depth_delta;
    r = rgb_residual(a, g_ops.state, g_ops.ipartials, 0, st(s)); if (r) return r;
    int res[2];
    KT_CUDA(cudaMemcpyAsync(res, (char*)g_ops.state + offsetof(OdomState, rgb_count), 2 * sizeof(int), cudaMemcpyDeviceToHost, st(s)));
    KT_CUDA(cudaStreamSynchronize(st(s)));
    *count = res[0]; *sigma_sum = res[1];
    return KT_OK;
}

int kt_op_generate_image(const float* vmap, const float* nmap, const uint8_t* vmap_curr_color, const float* light_pos3, int n_lights,
                         uint8_t* dst_rgb, uint8_t* dst_color_rgb, int rows, int cols, void* s)
{
    int r = generate_views(vmap, nmap, vmap_curr_color, rows, cols, light_pos3, n_lights, dst_rgb, dst_color_rgb, 0, 0, 0, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK;
}

int kt_op_generate_depth(const float* Rinv9, const float* t3, const float* vmap, const float* nmap, uint16_t* dst, int rows, int cols, float max_depth, void* s)
{
    (void)max_depth;                               // unused by the reference kernel too (image_generator.cu:187-211)
    int r = generate_views(vmap, nmap, 0, rows, cols, 0, 0, 0, 0, Rinv9, t3, dst, st(s)); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(st(s))); return KT_OK;
}

int kt_op_rgb_step(const void* corres, float sigma, const float* cloud, float fx, float fy, const int16_t* dIdx, const int16_t* dIdy,
                   float sobel_scale, int rows, int cols, float* A_host, float* b_host, void* s)
{
    KT_OPS_LOCK();
    int r = ensure_scratch(); if (r) return r;
    RgbLevelArgs a; std::memset(&a, 0, sizeof(a));
    a.corres = const_cast<void*>(corres); a.cloud = cloud; a.fx = fx; a.fy = fy; a.dIdx = dIdx; a.dIdy = dIdy; a.sobel_scale = sobel_scale; a.rows = rows; a.cols = cols;
    r = rgb_iteration(a, g_ops.state, g_ops.partials, 0, 0, sigma, st(s)); if (r) return r;
    float sums[32];
    KT_CUDA(cudaMemcpyAsync(sums, (char*)g_ops.state + offsetof(OdomState, sums_rgb), 32 * sizeof(float), cudaMemcpyDeviceToHost, st(s)));
    KT_CUDA(cudaStreamSynchronize(st(s)));
    unpack_normal_equations(sums, A_host, b_host);
    return KT_OK;
}

} // extern "C"

// ---- place-recognition operators (kt_surf.cu, kt_place.cu, kt_slice.cu); synchronous ----
namespace {
// the operators' small integer scratch, kept between calls so that a call does not allocate
int place_ints(size_t n, int** out)
{
    int r = g_ops.place_ints.grow(n, n, "operator counts"); if (r) return r;
    *out = g_ops.place_ints.get();
    return 0;
}
}

extern "C" {

int kt_op_surf(const uint8_t* rgb, int rows, int cols, float thr, int max_features, float* kp, float* desc, int* n_out, void* s)
{
    if (!rgb || !kp || !desc || !n_out) { set_error("kt_op_surf: null argument"); return KT_ERR_INVALID; }
    KT_OPS_LOCK();
    int* n_dev = 0; int r;
    if ((r = place_ints(1, &n_dev))) return r;
    if ((r = surf(rgb, rows, cols, thr, max_features, kp, desc, n_dev, &g_ops.surf_ws, st(s)))) return r;
    KT_CUDA(cudaMemcpyAsync(n_out, n_dev, sizeof(int), cudaMemcpyDeviceToHost, st(s)));
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_keypoints_3d(const float* kp, int n, const uint16_t* depth, int rows, int cols, const float* k4, float* xyz, void* s)
{
    if (!kp || !depth || !k4 || !xyz || n < 0 || rows <= 0 || cols <= 0) { set_error("kt_op_keypoints_3d: bad argument"); return KT_ERR_INVALID; }
    if (n == 0) return KT_OK;
    KT_OPS_LOCK();
    int* n_dev = 0; int r;
    if ((r = place_ints(1, &n_dev))) return r;
    KT_CUDA(cudaMemcpyAsync(n_dev, &n, sizeof(int), cudaMemcpyHostToDevice, st(s)));
    if ((r = keypoints_3d(kp, n_dev, n, depth, rows, cols, intr4(k4), xyz, st(s)))) return r;
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_match_ratio(const float* db, int n_seg, int stride, const int* seg_counts, const float* q, int n_query, float ratio, int* best, float* d1,
                      float* d2, uint8_t* pass, int* seg_passes, void* s)
{
    if (!db || !q || !best || !d1 || !d2 || !pass || n_seg < 0 || stride < 0 || n_query < 0) { set_error("kt_op_match_ratio: bad argument"); return KT_ERR_INVALID; }
    if (n_seg == 0 || stride == 0) return KT_OK;
    KT_OPS_LOCK();
    int* ints = 0; int r;
    if ((r = place_ints(2 * (size_t)n_seg + 1, &ints))) return r;
    std::vector<int> h((size_t)n_seg + 1, stride);
    if (seg_counts) for (int g = 0; g < n_seg; ++g) h[(size_t)g] = std::max(0, std::min(stride, seg_counts[g]));
    h[(size_t)n_seg] = n_query;
    KT_CUDA(cudaMemcpyAsync(ints, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, st(s)));
    if ((r = match_ratio(db, n_seg, stride, ints, q, ints + n_seg, n_query, ratio, best, d1, d2, pass, seg_passes ? ints + n_seg + 1 : 0, st(s)))) return r;
    if (seg_passes) KT_CUDA(cudaMemcpyAsync(seg_passes, ints + n_seg + 1, (size_t)n_seg * sizeof(int), cudaMemcpyDeviceToHost, st(s)));
    KT_CUDA(cudaStreamSynchronize(st(s)));
    return KT_OK;
}

int kt_op_pnp_ransac(const float* p_new, const float* p_old, const float* uv_old, int n, const float* k4, int iterations, float thr, uint64_t seed,
                     double* pose12, uint8_t* inliers, int* n_inliers)
{
    if (!p_new || !p_old || !uv_old || !k4 || !pose12 || !inliers || !n_inliers || n < 3 || iterations < 1) { set_error("kt_op_pnp_ransac: bad argument"); return KT_ERR_INVALID; }
    KT_OPS_LOCK();
    Allocations b; const char* W = "kt_op_pnp_ransac scratch";
    float *pn, *po, *uv; double* pose; unsigned char* in; int* ni; int r;
    if ((r = b.device(&pn, 3 * (size_t)n, W)) || (r = b.device(&po, 3 * (size_t)n, W)) || (r = b.device(&uv, 2 * (size_t)n, W)) || (r = b.device(&pose, 12, W)) ||
        (r = b.device(&in, (size_t)n, W)) || (r = b.device(&ni, 1, W))) return r;
    KT_CUDA(cudaMemcpy(pn, p_new, 12 * (size_t)n, cudaMemcpyHostToDevice));
    KT_CUDA(cudaMemcpy(po, p_old, 12 * (size_t)n, cudaMemcpyHostToDevice));
    KT_CUDA(cudaMemcpy(uv, uv_old, 8 * (size_t)n, cudaMemcpyHostToDevice));
    PnpArgs a; a.p_new = pn; a.p_old = po; a.uv_old = uv; a.n = n; a.k = intr4(k4); a.iterations = iterations; a.threshold_px = thr; a.seed = seed;
    if ((r = pnp_ransac(a, &g_ops.pnp_ws, pose, in, ni, 0))) return r;
    KT_CUDA(cudaMemcpy(pose12, pose, 12 * sizeof(double), cudaMemcpyDeviceToHost));
    KT_CUDA(cudaMemcpy(inliers, in, (size_t)n, cudaMemcpyDeviceToHost));
    KT_CUDA(cudaMemcpy(n_inliers, ni, sizeof(int), cudaMemcpyDeviceToHost));
    return KT_OK;
}

int kt_op_cloud_fitness(const uint16_t* src_depth, const uint16_t* dst_depth, int rows, int cols, const float* k4, float leaf, const float* T12,
                        double* fitness, size_t* n_src, size_t* n_dst)
{
    if (!src_depth || !dst_depth || !k4 || !T12 || !fitness || !n_src || !n_dst || rows <= 0 || cols <= 0) { set_error("kt_op_cloud_fitness: bad argument"); return KT_ERR_INVALID; }
    KT_OPS_LOCK();
    const size_t P = (size_t)rows * cols;
    Allocations b; const char* W = "kt_op_cloud_fitness scratch";
    kt_point_xyzrgb *cs, *cd; kt_point_xyzrgbnormal *os, *od; double* d2; int r;
    if ((r = b.device(&cs, P, W)) || (r = b.device(&cd, P, W)) || (r = b.device(&os, P, W)) || (r = b.device(&od, P, W)) || (r = b.device(&d2, P + 8, W))) return r;
    if ((r = depth_to_cloud(src_depth, rows, cols, intr4(k4), cs, 0)) || (r = depth_to_cloud(dst_depth, rows, cols, intr4(k4), cd, 0))) return r;
    return cloud_fitness(cs, P, cd, P, leaf, T12, &g_ops.slice_ws, &g_ops.fit_ws, os, od, P, d2, fitness, n_src, n_dst, 0);
}

} // extern "C"
