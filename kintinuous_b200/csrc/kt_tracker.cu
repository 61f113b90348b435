// kintinuous_b200 -- the per-frame orchestrator behind kt_process_frame.
//
// Replaces (reference, src/frontend/): KintinuousTracker::{ctor, reset, processFrame, finalise, vWrapCopyUpdate,
// mutexOutCloudBuffer} (KintinuousTracker.cpp:71-182, 262-354, 444-915, 1003-1048, 1075-1085, 1156-1208),
// TsdfVolume (TSDFVolume.cpp:60-172), ColorVolume, and the drivers ICPOdometry::getIncrementalTransformation
// (ICPOdometry.cpp:68-186) / RGBDOdometry::getIncrementalTransformation (RGBDOdometry.cpp:165-393).
//
// Design (DESIGN.md section 3): everything of a frame is enqueued on ONE stream with exactly one host
// synchronisation -- after the odometry, because the shift decision and the slice hand-off are host logic in
// the reference too.  The reference's frame has 59 launches, 26 cudaDeviceSynchronize and 19 blocking D2H
// copies; here: 6 front-end launches (bilateral, 3 pyrDown, maps, colour prep), ONE cooperative odometry launch (all levels and
// iterations, solve on device), 3 fusion launches (scaleDepth, z table, integrate), 1 raycast launch that also builds the model
// pyramid, one 48-byte D2H.  kt_prefetch_frame builds the NEXT frame's front end on a side stream into a spare buffer set while the
// current frame is being fused.  The CUDA-free bookkeeping of the shifting volume lives in kt_shift.hpp (CPU-tested).
#include "kt_ops.h"
#include "kt_shift.hpp"
#include "kt_posegraph.hpp"
#include "kt_deform.hpp"
#include "kt_pgo.hpp"
#include <cstdlib>
#include "../../include/kintinuous_b200.h"
#include <vector>
#include <unordered_map>
#include <cstring>
#include <cmath>
#include <climits>
#include <algorithm>
#include <cstdarg>
#include <cstdio>

namespace kt {

// ---- error plumbing ------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
std::atomic<long long> g_launches(0);
void set_error(const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}
const char* last_error() { return g_err; }
int cuda_check(cudaError_t e, const char* what, const char* file, int line)
{
    if (e == cudaSuccess) return 0;
    set_error("CUDA error '%s' at %s:%d (%s)", cudaGetErrorString(e), file, line, what);
    return KT_ERR_CUDA;
}

DeviceInfo& device_info()
{
    enum { MAXD = 64 };
    static DeviceInfo info[MAXD];
    static std::atomic<int> ready[MAXD];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAXD) dev = 0;
    if (!ready[dev].load(std::memory_order_acquire)) {
        DeviceInfo d; d.sm_count = 0; d.smem_optin = 0; d.configured = 0;
        cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&d.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (d.sm_count <= 0) d.sm_count = 132;
        info[dev] = d;
        ready[dev].store(1, std::memory_order_release);
    }
    return info[dev];
}

// ---- small host math (what the reference takes from Eigen) ---------------------------------------
struct M3 { float m[9]; };
struct V3 { float v[3]; };
static M3 m3_identity() { M3 r = {{1, 0, 0, 0, 1, 0, 0, 0, 1}}; return r; }
static M3 m3_inverse(const M3& a)      // Eigen::Matrix3f::inverse(): cofactors / determinant
{
    const float* m = a.m;
    auto M = [&](int i, int j) { return m[i * 3 + j]; };
    auto cof = [&](int i, int j) { return M((i + 1) % 3, (j + 1) % 3) * M((i + 2) % 3, (j + 2) % 3) - M((i + 1) % 3, (j + 2) % 3) * M((i + 2) % 3, (j + 1) % 3); };
    float c00 = cof(0, 0), c10 = cof(1, 0), c20 = cof(2, 0);
    float det = (c00 * M(0, 0) + c10 * M(1, 0)) + c20 * M(2, 0);
    float invdet = 1.0f / det;
    M3 r;
    r.m[0] = c00 * invdet; r.m[1] = c10 * invdet; r.m[2] = c20 * invdet;
    r.m[3] = cof(0, 1) * invdet; r.m[4] = cof(1, 1) * invdet; r.m[5] = cof(2, 1) * invdet;
    r.m[6] = cof(0, 2) * invdet; r.m[7] = cof(1, 2) * invdet; r.m[8] = cof(2, 2) * invdet;
    return r;
}
static Mat33 to_mat33(const float* m) { Mat33 r; r.r0 = make_float3(m[0], m[1], m[2]); r.r1 = make_float3(m[3], m[4], m[5]); r.r2 = make_float3(m[6], m[7], m[8]); return r; }

// A slice lives in PINNED host memory carved from the context's arena; its device -> host copy is asynchronous (side stream) and
// `ready` fires when the bytes have landed.  The reference downloads into a pageable std::vector with a blocking cudaMemcpy inside
// processFrame (KintinuousTracker.cpp:1166, containers/device_memory.cpp:146-157).
struct SliceRec { int dimension; kt_point_xyzrgb* points; size_t count; kt_point_xyzrgbnormal* processed; size_t processed_count; bool has_processed;
                  kt_mesh_vertex* mesh_verts; uint32_t* mesh_tris; size_t mesh_nv, mesh_nt; bool has_mesh;
                  cudaEvent_t ready; float camera_t[3]; float camera_R[9]; uint64_t utime; };

// Pinned host memory handed out in slabs (one cudaHostAlloc per 64 MB, not per slice); everything is released together by kt_reset.
struct PinnedArena {
    std::vector<std::pair<char*, size_t> > chunks; size_t chunk_used; size_t current;
    PinnedArena() : chunk_used(0), current(0) {}
    void* alloc(size_t bytes)
    {
        bytes = (bytes + 255) & ~(size_t)255;
        while (current < chunks.size() && chunk_used + bytes > chunks[current].second) { ++current; chunk_used = 0; }
        if (current >= chunks.size()) {
            const size_t sz = std::max(bytes, (size_t)64 << 20);
            void* q = 0;
            if (cudaHostAlloc(&q, sz, cudaHostAllocDefault) != cudaSuccess) return 0;
            chunks.push_back(std::make_pair((char*)q, sz));
            current = chunks.size() - 1; chunk_used = 0;
        }
        void* r = chunks[current].first + chunk_used;
        chunk_used += bytes;
        return r;
    }
    void rewind() { current = 0; chunk_used = 0; }
    void release() { for (auto& c : chunks) cudaFreeHost(c.first); chunks.clear(); rewind(); }
};

// what the host reads back after the odometry of a frame
struct OdomResult { float Rcurr[9]; float tcurr[3]; int timeout; unsigned int seq; int pad[2]; };     // seq: written last by the odometry kernel (mapped host memory)

} // namespace kt

using namespace kt;

struct kt_ctx {
    kt_config cfg;
    cudaStream_t stream, stream2;          // stream2: pose-independent side work (scaleDepth) overlapped with the pyramid / ICP
    cudaEvent_t ev_input, ev_scaled;
    float size, voxel, trunc;
    float volumeBasis[3], currentGlobalCamera[3];
    int voxelWrap[3];
    int global_time; uint64_t current_utime;
    int overlap, parked;
    std::vector<M3> rmats; std::vector<V3> tvecs;
    std::vector<SliceRec> slices;
    std::vector<kt_dense_pose> dense_poses;      // densePoseGraph (KintinuousTracker.h:171)
    FILE* pose_log;                              // <saveFile>.poses (outputPose)
    int iterations[LEVELS];
    // device memory
    int16_t* tsdf; uint8_t* color;
    uint16_t* depth_raw; uint8_t* rgb;
    // double-buffered inputs: kt_prefetch_frame fills the spare set on a copy stream while the previous frame is still being fused
    uint16_t* depth_alt; uint8_t* rgb_alt; const void* pf_depth; const void* pf_rgb; bool pf_valid;
    // ... and the pose-independent front end of the NEXT frame (scaleDepth, bilateral, pyrDown, vertex / normal maps) is built into a
    // spare set on the same side stream, so that it overlaps the integrate / ray-cast of the frame before (they leave issue slots idle)
    uint16_t* depths_alt[LEVELS]; float* vmaps_alt[LEVELS]; float* nmaps_alt[LEVELS]; float* depth_scaled_alt;
    bool pf_built;             // the prefetched set holds the finished front end
    bool color_prepared;       // cw_scratch / rgbf_scratch hold this frame's per-pixel colour inputs
    bool frontend_ready;       // set for the duration of one process_frame_device call
    cudaStream_t stream_copy; cudaEvent_t ev_prefetch, ev_done[2], ev_maps; int last_parity; bool maps_on_stream;   // ev_maps: this frame's front end (on `stream`) has written the current maps
    uint16_t* depths_curr[LEVELS];
    float* vmaps_g_prev[LEVELS]; float* nmaps_g_prev[LEVELS]; float* vmaps_curr[LEVELS]; float* nmaps_curr[LEVELS];
    uint8_t* vmap_curr_color; float* depth_scaled; float* ztable; float* cw_scratch; float* rgbf_scratch; float* cw_alt; float* rgbf_alt;
    unsigned long long* xwords_dev; bool xwords_clean;      // exchange words of the whole-frame odometry kernels; zero between frames
    OdomState* state; float* partials; int* ipartials; float* trace_dev; float* pose12_dev; unsigned int* bar_dev; unsigned int bar_count; long long* prof_dev;
    kt_point_xyzrgb* cloud_dev; unsigned int* counter_dev; size_t cloud_capacity; size_t cloud_count;
    // slice hand-off: pinned arena, asynchronous download on stream_slices; ev_cloud_free = the last download has left cloud_dev / proc_dev
    PinnedArena* slice_arena; cudaStream_t stream_slices; cudaEvent_t ev_cloud_ready, ev_cloud_free; bool cloud_busy;
    // CloudSliceProcessor on the device (kt_slice.cu): weight cull + voxel grid + normals of every slice before it leaves the GPU
    int slice_processing, slice_weight_cull; SliceWorkspace slice_ws; kt_point_xyzrgbnormal* proc_dev; size_t proc_count;
    // marching cubes of every slice's box before it is cleared (kt_mesh.cu); buffers grow at a shift, downloaded with the slice
    int slice_meshing, mesh_weight_cull; MeshWorkspace mesh_ws; kt_mesh_vertex* mesh_verts_dev; uint32_t* mesh_tris_dev;
    size_t mesh_verts_cap, mesh_tris_cap, mesh_nv, mesh_nt;
    // the map as deformed by the last kt_deform_map (kt_deform.cu): one record per slice recorded before that call, in its own pinned
    // arena, or the slice's own buffers when the call left the map unchanged
    struct Deformed { kt_point_xyzrgbnormal* processed; kt_mesh_vertex* mesh_verts; };
    std::vector<Deformed> deformed; PinnedArena* deform_arena;
    // loop closure (kt_close_loop, kt_pgo.cu): the accepted loops with their inliers, and the optimised nodes of the last accepted one
    struct Loop { uint64_t time1, time2; double C[16]; std::vector<float> in1, in2; };
    std::vector<Loop> loops; std::vector<kt_dense_pose> pgo_nodes;
    // RGB-D
    float* lastDepth[LEVELS]; float* nextDepth[LEVELS]; uint8_t* lastImage[LEVELS]; uint8_t* nextImage[LEVELS];
    int16_t* nextdIdx[LEVELS]; int16_t* nextdIdy[LEVELS]; float* pointClouds[LEVELS]; void* corresImg[LEVELS];
    // pinned host staging
    float* pose12_host; OdomResult* result_host; float* result_dev_alias; unsigned int pose_seq; bool pose_spin; float* trace_host; unsigned int* counter_host;
    int trace_iters; int shifted_last;
    // timing
    bool timing; cudaEvent_t ev[7]; float stage_ms[6]; cudaEvent_t ev_icp[2]; cudaEvent_t ev_krn[4]; cudaEvent_t ev_span[2];     // ev_krn: integrate / raycast launches alone (without the cross-GPU barriers the stage timers include)
    long long launches_at_create;
    std::vector<void*> allocs;
    // ONE volume shared by `world` GPUs (one process per GPU; peers' arenas are mapped through CUDA IPC): TSDF plane replicated, colour /
    // weight plane sharded block-cyclically by storage z (VolumeView, kt_ops.h)
    int world, rank, local_planes, mg_block;
    uint8_t* arena; size_t arena_bytes;
    size_t off_tsdf, off_color, off_vmap[LEVELS], off_nmap[LEVELS], off_vcol, off_flags, off_xwords;
    bool split_icp;            // KT_MG_SPLIT_ICP: pixel rows of the ICP split over the ranks, normal equations all-reduced in the kernel over peer memory
    uint8_t* peer_arena[MAX_GPUS]; bool connected;
    unsigned int** peer_flags_dev; unsigned int epoch; int* mg_error_dev; int* mg_error_host;
    VolumeView vv;
    float last_int_Rinv[9], last_int_t[3]; int last_int_wrap[3];       // arguments of the last integration (kt_debug_last_integrate)
    uint8_t* view_dev;                                                  // GUI taps: shaded image, colour image, model depth (allocated on first use)
};

namespace {

const int MAX_TRACE_ITERS = 64;

template <class T> int dev_alloc(kt_ctx* c, T** p, size_t count)
{
    void* q = 0;
    const size_t bytes = count * sizeof(T);
    KT_CUDA(cudaMalloc(&q, bytes ? bytes : 1));
    c->allocs.push_back(q);
    *p = (T*)q;
    return 0;
}

void vwrap_copy(const kt_ctx* c, int* w)       // KintinuousTracker::vWrapCopyUpdate (.cpp:1075-1085)
{
    vwrap_nonneg(c->voxelWrap, c->cfg.vol, w);
}

int fetch_cloud(kt_ctx* c, const int* vWrapCopy, const int* lo, const int* hi)      // TsdfVolume::fetchCloud (TSDFVolume.cpp:131-172)
{
    // the previous slice's asynchronous download may still be reading cloud_dev
    if (c->cloud_busy) { KT_CUDA(cudaStreamWaitEvent(c->stream, c->ev_cloud_free, 0)); c->cloud_busy = false; }
    KT_CUDA(cudaMemsetAsync(c->counter_dev, 0, sizeof(unsigned int), c->stream));
    float3 vs = make_float3(c->size, c->size, c->size);
    int r = c->world > 1
        ? extract_slice_mg(c->vv, vs, c->cfg.vol, c->cloud_dev, c->cloud_capacity, make_int3(vWrapCopy[0], vWrapCopy[1], vWrapCopy[2]),
                           lo[0], hi[0], lo[1], hi[1], lo[2], hi[2], 1, make_int3(c->voxelWrap[0], c->voxelWrap[1], c->voxelWrap[2]), c->counter_dev, c->stream)
        : extract_slice(c->tsdf, vs, c->cfg.vol, c->cloud_dev, c->cloud_capacity, make_int3(vWrapCopy[0], vWrapCopy[1], vWrapCopy[2]), c->color,
                        lo[0], hi[0], lo[1], hi[1], lo[2], hi[2], 1, make_int3(c->voxelWrap[0], c->voxelWrap[1], c->voxelWrap[2]), c->counter_dev, c->stream);
    if (r) return r;
    KT_CUDA(cudaMemcpyAsync(c->counter_host, c->counter_dev, sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(cudaStreamSynchronize(c->stream));
    c->cloud_count = std::min((size_t)*c->counter_host, c->cloud_capacity);
    return 0;
}

// Marching cubes over the box [lo, hi) that fetch_cloud has just extracted, on the tracker stream and before the box is cleared, into
// the context's mesh buffers (grown here: the count is read back first, once).  MeshGenerator::calculateMesh (MeshGenerator.cpp:193-227)
// on the device, by a different algorithm (kt_mesh.cu).
int mesh_box(kt_ctx* c, const int* vWrapCopy, const int* lo, const int* hi)
{
    // the previous slice's asynchronous download may still be reading the mesh buffers
    if (c->cloud_busy) { KT_CUDA(cudaStreamWaitEvent(c->stream, c->ev_cloud_free, 0)); c->cloud_busy = false; }
    MeshArgs a;
    a.tsdf = c->tsdf; a.color = c->color; a.vol = c->cfg.vol; a.volume_size = make_float3(c->size, c->size, c->size);
    a.wrap = make_int3(vWrapCopy[0], vWrapCopy[1], vWrapCopy[2]); a.real_wrap = make_int3(c->voxelWrap[0], c->voxelWrap[1], c->voxelWrap[2]);
    a.minX = lo[0]; a.maxX = hi[0]; a.minY = lo[1]; a.maxY = hi[1]; a.minZ = lo[2]; a.maxZ = hi[2]; a.weight_cull = c->mesh_weight_cull;
    size_t nv = 0, nt = 0;
    int r = mesh_count(a, &c->mesh_ws, &nv, &nt, c->stream); if (r) return r;
    if (nv > c->mesh_verts_cap || nt > c->mesh_tris_cap) {
        KT_CUDA(cudaStreamSynchronize(c->stream_slices));
        if (nv > c->mesh_verts_cap) {
            if (c->mesh_verts_dev) cudaFree(c->mesh_verts_dev);
            c->mesh_verts_dev = 0; c->mesh_verts_cap = 0;
            const size_t want = nv + nv / 4 + 1024;
            KT_CUDA(cudaMalloc((void**)&c->mesh_verts_dev, want * sizeof(kt_mesh_vertex)));
            c->mesh_verts_cap = want;
        }
        if (nt > c->mesh_tris_cap) {
            if (c->mesh_tris_dev) cudaFree(c->mesh_tris_dev);
            c->mesh_tris_dev = 0; c->mesh_tris_cap = 0;
            const size_t want = nt + nt / 4 + 1024;
            KT_CUDA(cudaMalloc((void**)&c->mesh_tris_dev, want * 3 * sizeof(uint32_t)));
            c->mesh_tris_cap = want;
        }
    }
    r = mesh_emit(a, &c->mesh_ws, nv, c->mesh_verts_dev, c->mesh_tris_dev, c->stream); if (r) return r;
    c->mesh_nv = nv; c->mesh_nt = nt;
    return 0;
}

// mutexOutCloudBuffer (KintinuousTracker.cpp:1156-1208): record the extracted cloud as a CloudSlice.  The points go to pinned host
// memory with an ASYNCHRONOUS copy on a side stream -- the frame's clear / integrate / ray cast do not wait for it; readers of the slice
// do (kt_get_slice waits on the slice's event).  With slice processing on, the slice is culled, voxel-gridded and given normals on the
// device first (kt_slice.cu) and both clouds are handed out.
int push_slice(kt_ctx* c, int dimension)
{
    SliceRec s; s.dimension = dimension; s.points = 0; s.count = c->cloud_count; s.processed = 0; s.processed_count = 0; s.has_processed = false; s.ready = 0;
    s.has_mesh = c->slice_meshing != 0; s.mesh_verts = 0; s.mesh_tris = 0;
    s.mesh_nv = s.has_mesh ? c->mesh_nv : 0; s.mesh_nt = s.has_mesh ? c->mesh_nt : 0;
    c->proc_count = 0;
    if (c->slice_processing && c->cloud_count) {
        if (!c->proc_dev) { void* q = 0; KT_CUDA(cudaMalloc(&q, c->cloud_capacity * sizeof(kt_point_xyzrgbnormal))); c->allocs.push_back(q); c->proc_dev = (kt_point_xyzrgbnormal*)q; }
        int r = process_slice(c->cloud_dev, c->cloud_count, c->slice_weight_cull, c->voxel, 20, c->proc_dev, c->cloud_capacity, &c->proc_count, &c->slice_ws, c->stream);
        if (r) return r;
    }
    s.has_processed = c->slice_processing != 0;
    s.processed_count = c->proc_count;
    if (c->cloud_count || s.mesh_nv) {
        if (c->cloud_count) s.points = (kt_point_xyzrgb*)c->slice_arena->alloc(c->cloud_count * sizeof(kt_point_xyzrgb));
        if (c->proc_count) s.processed = (kt_point_xyzrgbnormal*)c->slice_arena->alloc(c->proc_count * sizeof(kt_point_xyzrgbnormal));
        if (s.mesh_nv) s.mesh_verts = (kt_mesh_vertex*)c->slice_arena->alloc(s.mesh_nv * sizeof(kt_mesh_vertex));
        if (s.mesh_nt) s.mesh_tris = (uint32_t*)c->slice_arena->alloc(s.mesh_nt * 3 * sizeof(uint32_t));
        if ((c->cloud_count && !s.points) || (c->proc_count && !s.processed) || (s.mesh_nv && !s.mesh_verts) || (s.mesh_nt && !s.mesh_tris)) {
            set_error("pinned host memory for a slice of %zu points", c->cloud_count); return KT_ERR_CUDA;
        }
        KT_CUDA(cudaEventCreateWithFlags(&s.ready, cudaEventDisableTiming));
        KT_CUDA(cudaEventRecord(c->ev_cloud_ready, c->stream));
        KT_CUDA(cudaStreamWaitEvent(c->stream_slices, c->ev_cloud_ready, 0));
        if (c->cloud_count) KT_CUDA(cudaMemcpyAsync(s.points, c->cloud_dev, c->cloud_count * sizeof(kt_point_xyzrgb), cudaMemcpyDeviceToHost, c->stream_slices));
        if (c->proc_count) KT_CUDA(cudaMemcpyAsync(s.processed, c->proc_dev, c->proc_count * sizeof(kt_point_xyzrgbnormal), cudaMemcpyDeviceToHost, c->stream_slices));
        if (s.mesh_nv) KT_CUDA(cudaMemcpyAsync(s.mesh_verts, c->mesh_verts_dev, s.mesh_nv * sizeof(kt_mesh_vertex), cudaMemcpyDeviceToHost, c->stream_slices));
        if (s.mesh_nt) KT_CUDA(cudaMemcpyAsync(s.mesh_tris, c->mesh_tris_dev, s.mesh_nt * 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream_slices));
        KT_CUDA(cudaEventRecord(s.ready, c->stream_slices));
        KT_CUDA(cudaEventRecord(c->ev_cloud_free, c->stream_slices));
        c->cloud_busy = true;
    }
    for (int i = 0; i < 3; ++i) s.camera_t[i] = c->currentGlobalCamera[i];
    for (int i = 0; i < 9; ++i) s.camera_R[i] = c->rmats.back().m[i];
    s.utime = c->current_utime;
    c->slices.push_back(s);
    return 0;
}

void drop_slices(kt_ctx* c)
{
    if (c->stream_slices) cudaStreamSynchronize(c->stream_slices);
    for (auto& s : c->slices) if (s.ready) cudaEventDestroy(s.ready);
    c->slices.clear();
    if (c->slice_arena) c->slice_arena->rewind();
    c->cloud_busy = false;
}

int do_integrate(kt_ctx* c, const M3& Rinv, const V3& t, const int* wrap)
{
    const int rows = c->cfg.rows, cols = c->cfg.cols;
    Intr k = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    IntegrateArgs a;
    a.depth_scaled = c->depth_scaled; a.rows = rows; a.cols = cols; a.k = k; a.volume_size = make_float3(c->size, c->size, c->size);
    a.Rinv = to_mat33(Rinv.m); a.t = make_float3(t.v[0], t.v[1], t.v[2]); a.trunc = c->trunc;
    a.tsdf = c->tsdf; a.color = c->color; a.vol = c->cfg.vol; a.wrap = make_int3(wrap[0], wrap[1], wrap[2]);
    a.rgb = c->rgb; a.nmap_curr = c->nmaps_curr[0]; a.angle_color = c->cfg.angle_color != 0;
    for (int k = 0; k < 9; ++k) c->last_int_Rinv[k] = Rinv.m[k];
    for (int k = 0; k < 3; ++k) { c->last_int_t[k] = t.v[k]; c->last_int_wrap[k] = wrap[k]; }
    a.reset_words = c->xwords_dev; a.reset_count = odom_exchange_used(&a.reset_stride); c->xwords_clean = true;       // the prologue launch of integrate() zeroes them
    a.multi = c->world > 1 ? 1 : 0; a.vv = c->vv; a.cw = c->color_prepared ? c->cw_scratch : 0; a.rgbf = c->color_prepared ? (float4*)c->rgbf_scratch : 0;
    return integrate(a, c->ztable, c->stream);
}

int run_odometry(kt_ctx* c, const M3& Rprev, const V3& tprev, M3* Rcurr, V3* tcurr)
{
    const int rows = c->cfg.rows, cols = c->cfg.cols;
    const int mode = c->cfg.odometry;
    int r;
    for (int k = 0; k < 9; ++k) c->pose12_host[k] = Rprev.m[k];
    for (int k = 0; k < 3; ++k) c->pose12_host[9 + k] = tprev.v[k];
    const float distThres = 0.10f, angleThres = sinf(20.f * 3.14159254f / 180.f);      // ICPOdometry.h:35-36
    Intr K = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    int total_iters = 0;
    // KT_FORCE_PER_ITERATION (test hook): take the per-iteration kernels -- the path of images too large for the whole-frame kernels'
    // shared-memory stage -- on an image that would fit, so that it can be compared against the whole-frame path and the reference
    static const bool force_per_iteration = getenv("KT_FORCE_PER_ITERATION") != nullptr;
    if (mode == 0 && !force_per_iteration) {
        // ICP-only: the whole coarse-to-fine loop is ONE cooperative launch (kt_icp.cu, icp_frame_kernel)
        IcpLevelArgs la[LEVELS];
        for (int level = 0; level < LEVELS; ++level) {
            IcpLevelArgs ia = {c->vmaps_curr[level], c->nmaps_curr[level], c->vmaps_g_prev[level], c->nmaps_g_prev[level], rows >> level, cols >> level,
                               intr_level(K, level), distThres, angleThres};
            la[level] = ia;
            total_iters += c->iterations[level];
        }
        if (c->timing) cudaEventRecord(c->ev_icp[0], c->stream);
        if (!c->xwords_clean && (r = odom_exchange_reset(c->xwords_dev, c->stream))) return r;
        c->xwords_clean = false;
        ++c->pose_seq;
        unsigned long long* peers[MAX_GPUS];
        for (int g = 0; g < MAX_GPUS; ++g) peers[g] = (unsigned long long*)(c->peer_arena[g] + c->off_xwords);
        if ((r = icp_frame(la, c->iterations, c->pose12_host, c->state, c->xwords_dev, c->trace_dev, &c->state->odo_timeout, c->timing ? c->prof_dev : 0,
                           c->pose_spin ? c->result_dev_alias : 0, c->pose_seq, c->stream, c->split_icp ? peers : 0, c->world, c->rank))) return r;
        if (c->timing) cudaEventRecord(c->ev_icp[1], c->stream);
    }
    const double SOBEL_SCALE = 1.0 / std::pow(2.0, 3);
    const int minimumGradientMagnitudes[4] = {12, 5, 3, 1};
    bool per_iteration_path = (mode != 0) || force_per_iteration;
    if (force_per_iteration) {
        KT_CUDA(cudaMemcpyAsync(c->pose12_dev, c->pose12_host, 12 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        if ((r = odom_begin_frame(c->state, c->pose12_dev, c->stream))) return r;
    } else if (mode != 0) {
        // whole-frame RGB-D / ICP+RGB-D kernel (kt_rgb.cu, rgbd_frame_kernel): ONE cooperative launch for all levels and iterations
        IcpLevelArgs la[LEVELS]; RgbLevelArgs ra4[LEVELS];
        for (int level = 0; level < LEVELS; ++level) {
            const int lr = rows >> level, lc = cols >> level;
            Intr kl = intr_level(K, level);
            IcpLevelArgs ia = {c->vmaps_curr[level], c->nmaps_curr[level], c->vmaps_g_prev[level], c->nmaps_g_prev[level], lr, lc, kl, distThres, angleThres};
            la[level] = ia;
            const int div = 1 << level;
            RgbLevelArgs& ra = ra4[level];
            ra.dIdx = c->nextdIdx[level]; ra.dIdy = c->nextdIdy[level]; ra.last_depth = c->lastDepth[level]; ra.next_depth = c->nextDepth[level];
            ra.last_image = c->lastImage[level]; ra.next_image = c->nextImage[level]; ra.corres = c->corresImg[level]; ra.cloud = c->pointClouds[level];
            ra.rows = lr; ra.cols = lc;
            ra.min_scale = (float)(std::pow((double)minimumGradientMagnitudes[level], 2.0) / std::pow(SOBEL_SCALE, 2.0));
            ra.max_depth_delta = 0.07f; ra.fx = kl.fx; ra.fy = kl.fy; ra.sobel_scale = (float)SOBEL_SCALE;
            ra.Kfx = (double)K.fx / div; ra.Kfy = (double)K.fy / div; ra.Kcx = (double)K.cx / div; ra.Kcy = (double)K.cy / div;
        }
        if (!c->xwords_clean && (r = odom_exchange_reset(c->xwords_dev, c->stream))) return r;
        ++c->pose_seq;
        r = rgbd_frame(la, ra4, c->iterations, mode == 2 ? 1 : 0, c->pose12_host, c->state, c->xwords_dev, c->trace_dev, &c->state->odo_timeout,
                       c->pose_spin ? c->result_dev_alias : 0, c->pose_seq, c->stream);
        if (r == 0) c->xwords_clean = false;
        if (r < 0) return r;
        if (r == 0) { per_iteration_path = false; for (int level = 0; level < LEVELS; ++level) total_iters += c->iterations[level]; }
        else {       // image too large for the shared-memory stage: per-iteration kernels
            KT_CUDA(cudaMemcpyAsync(c->pose12_dev, c->pose12_host, 12 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
            if ((r = odom_begin_frame(c->state, c->pose12_dev, c->stream))) return r;
        }
    }
    for (int level = LEVELS - 1; level >= 0 && per_iteration_path; --level) {
        const int lr = rows >> level, lc = cols >> level;
        Intr kl = intr_level(K, level);
        IcpLevelArgs ia = {c->vmaps_curr[level], c->nmaps_curr[level], c->vmaps_g_prev[level], c->nmaps_g_prev[level], lr, lc, kl, distThres, angleThres};
        RgbLevelArgs ra;
        if (mode != 0) {
            const int div = 1 << level;
            // IntrDoublePrecision built from the float Intr (RGBDOdometry.cpp:70-73), per-level division in double
            const double dfx = (double)K.fx / div, dfy = (double)K.fy / div, dcx = (double)K.cx / div, dcy = (double)K.cy / div;
            if ((r = project_to_point_cloud(c->lastDepth[level], c->pointClouds[level], lr, lc, dfx, dfy, dcx, dcy, c->stream))) return r;
            ra.dIdx = c->nextdIdx[level]; ra.dIdy = c->nextdIdy[level]; ra.last_depth = c->lastDepth[level]; ra.next_depth = c->nextDepth[level];
            ra.last_image = c->lastImage[level]; ra.next_image = c->nextImage[level]; ra.corres = c->corresImg[level]; ra.cloud = c->pointClouds[level];
            ra.rows = lr; ra.cols = lc;
            ra.min_scale = (float)(std::pow((double)minimumGradientMagnitudes[level], 2.0) / std::pow(SOBEL_SCALE, 2.0));
            ra.max_depth_delta = 0.07f; ra.fx = kl.fx; ra.fy = kl.fy; ra.sobel_scale = (float)SOBEL_SCALE;
            ra.Kfx = dfx; ra.Kfy = dfy; ra.Kcx = dcx; ra.Kcy = dcy;
        }
        for (int iter = 0; iter < c->iterations[level]; ++iter) {
            float* trace = (total_iters < MAX_TRACE_ITERS) ? c->trace_dev : 0;
            if (mode == 0) {
                if ((r = icp_iteration(ia, c->state, c->partials, trace, 1, c->stream))) return r;
            } else {
                if ((r = rgb_residual(ra, c->state, c->ipartials, 1, c->stream))) return r;
                if (mode == 2 && (r = icp_iteration(ia, c->state, c->partials, 0, 0, c->stream))) return r;
                if ((r = rgb_iteration(ra, c->state, c->partials, trace, mode == 2 ? 2 : 1, 0.f, c->stream))) return r;
            }
            ++total_iters;
        }
    }
    c->trace_iters = std::min(total_iters, MAX_TRACE_ITERS);
    // one 64-byte read-back of the estimate (+ the trace when someone asked for it later: it stays on the device)
    static_assert(offsetof(OdomState, odo_timeout) == offsetof(OdomState, Rcurr) + 12 * sizeof(float), "the time-out flag travels with the pose");
    bool got = false;
    if (c->pose_spin && !per_iteration_path && !c->timing) {
        // the whole-frame kernel wrote the estimate into mapped host memory and then its sequence number: poll it (a few microseconds
        // after the kernel's last store) instead of a D2H copy + stream synchronisation; bounded, then the ordinary path takes over
        volatile unsigned int* seq = &c->result_host->seq;
        for (long spins = 0; spins < 4000000L; ++spins) { if (*seq == c->pose_seq) { got = true; break; } }
        std::atomic_thread_fence(std::memory_order_acquire);
    }
    if (!got) {
        KT_CUDA(cudaMemcpyAsync(c->result_host->Rcurr, (char*)c->state + offsetof(OdomState, Rcurr), 13 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        KT_CUDA(cudaStreamSynchronize(c->stream));
    }
    // mapped host memory: a timed-out barrier kernel wrote it in place
    if (c->world > 1 && *(volatile int*)c->mg_error_host) { set_error("cross-GPU barrier timed out waiting for rank %d", *c->mg_error_host - 1); return KT_ERR_STATE; }
    if (c->result_host->timeout) {
        cudaMemsetAsync(&c->state->odo_timeout, 0, sizeof(int), c->stream);
        set_error("odometry kernel: a CTA never arrived at the grid-wide sum (bounded poll gave up)"); return KT_ERR_STATE;
    }
    for (int k = 0; k < 9; ++k) Rcurr->m[k] = c->result_host->Rcurr[k];
    for (int k = 0; k < 3; ++k) tcurr->v[k] = c->result_host->tcurr[k];
    if (mode != 0) {
        for (int i = 0; i < LEVELS; ++i) { std::swap(c->lastDepth[i], c->nextDepth[i]); std::swap(c->lastImage[i], c->nextImage[i]); }   // RGBDOdometry.cpp:377-381
        float dx = tcurr->v[0] - tprev.v[0], dy = tcurr->v[1] - tprev.v[1], dz = tcurr->v[2] - tprev.v[2];
        if (std::sqrt(dx * dx + dy * dy + dz * dz) > 0.3) { *Rcurr = Rprev; *tcurr = tprev; }                                               // :383-387
    }
    return 0;
}

int mg_barrier(kt_ctx* c)
{
    if (c->world <= 1) return 0;
    if (!c->connected) { set_error("multi-GPU context used before kt_mgpu_connect"); return KT_ERR_STATE; }
    ++c->epoch;
    return xgpu_barrier(c->peer_flags_dev, (unsigned int*)(c->arena + c->off_flags), c->rank, c->world, c->epoch, c->mg_error_dev, c->stream);
}

// Pose-independent front end of one frame in TWO launches (kt_frontend.cu): bilateral filter + scaleDepth, then the depth pyramid, the
// vertex / normal maps of all levels, the colour-integration inputs and -- for -r / -ri -- the photometric pyramids and gradients
// (RGBDOdometry::populateRGBDData / firstRun + computeDerivativeImages, RGBDOdometry.cpp:140-175) into depth_m / intensity.
// vstale / nstale: the previous frame's maps when the outputs are a spare set (Q7 staleness), else null.
int build_frontend(kt_ctx* c, const uint16_t* depth_raw, const uint8_t* rgb, float* depth_scaled, uint16_t* const* depths, float* const* vmaps, float* const* nmaps,
                   float* const* vstale, float* const* nstale, float* cw, float* rgbf, float* const* depth_m, uint8_t* const* intensity, cudaStream_t s)
{
    const int rows = c->cfg.rows, cols = c->cfg.cols, mode = c->cfg.odometry;
    int r;
    Intr K = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    const bool use_icp_maps = (mode == 0) || (mode == 2) || c->cfg.angle_color;        // KintinuousTracker.cpp:465 (Q10)
    if ((r = bilateral_scale(depth_raw, use_icp_maps ? depths[0] : 0, depth_scaled, rows, cols, K, c->cfg.angle_color != 0, s))) return r;
    FrontendArgs fa;
    fa.depth_f = use_icp_maps ? depths[0] : 0; fa.depth_raw = depth_raw; fa.rgb = rgb; fa.rows = rows; fa.cols = cols; fa.k = K;
    fa.depths = depths; fa.vmaps = use_icp_maps ? vmaps : 0; fa.nmaps = use_icp_maps ? nmaps : 0; fa.vstale = vstale; fa.nstale = nstale;
    fa.cw = use_icp_maps ? cw : 0; fa.rgbf = use_icp_maps ? (float4*)rgbf : 0; fa.angle_color = c->cfg.angle_color != 0;
    fa.cut_off = (int)(6.0 * 1000);                                                      // RGBDOdometry.cpp:147
    fa.depth_m = depth_m; fa.intensity = intensity; fa.dIdx = depth_m ? c->nextdIdx : 0; fa.dIdy = depth_m ? c->nextdIdy : 0;
    if (use_icp_maps || depth_m) { if ((r = frontend_pyramid(fa, s))) return r; }
    c->color_prepared = use_icp_maps;
    return 0;
}

// densePoseGraph.push_back(DensePose(current_utime, [Rcurr | currentGlobalCamera], isLoopPose)); latestDensePoseId++ and, for tracked
// frames, outputPose (KintinuousTracker.cpp:529-536, :901-914)
void record_dense_pose(kt_ctx* c, bool first)
{
    kt_dense_pose d;
    d.timestamp = c->current_utime; d.is_loop_pose = first ? 1 : 0;
    const M3& R = c->rmats.back();
    for (int r = 0; r < 3; ++r) { for (int k = 0; k < 3; ++k) d.pose[r * 4 + k] = R.m[r * 3 + k]; d.pose[r * 4 + 3] = c->currentGlobalCamera[r]; }
    d.pose[12] = d.pose[13] = d.pose[14] = 0.f; d.pose[15] = 1.f;
    c->dense_poses.push_back(d);
    if (!first && c->pose_log) {
        char line[256];
        const int n = format_pose_line(c->current_utime, c->currentGlobalCamera, R.m, line, sizeof(line));
        if (n > 0) { fwrite(line, 1, (size_t)n, c->pose_log); fflush(c->pose_log); }
    }
}

void mark(kt_ctx* c, int i) { if (c->timing) cudaEventRecord(c->ev[i], c->stream); }

int process_frame_device(kt_ctx* c, uint64_t utime, kt_pose* out)
{
    const int rows = c->cfg.rows, cols = c->cfg.cols, V = c->cfg.vol;
    const int mode = c->cfg.odometry;
    int r;
    c->shifted_last = 0;
    mark(c, 0);
    if (!c->frontend_ready) {
        // the first frame's photometric pyramids are the "last" set (RGBDOdometry::firstRun), every later frame's the "next" set
        float* const* dm = mode != 0 ? (c->global_time == 0 ? c->lastDepth : c->nextDepth) : 0;
        uint8_t* const* im = mode != 0 ? (c->global_time == 0 ? c->lastImage : c->nextImage) : 0;
        if ((r = build_frontend(c, c->depth_raw, c->rgb, c->depth_scaled, c->depths_curr, c->vmaps_curr, c->nmaps_curr, 0, 0, c->cw_scratch, c->rgbf_scratch, dm, im, c->stream))) return r;
        // the look-ahead front end of the NEXT frame (kt_prefetch_frame, side stream) reads these maps as its stale-plane source (Q7)
        KT_CUDA(cudaEventRecord(c->ev_maps, c->stream));
        c->maps_on_stream = true;
    } else c->maps_on_stream = false;          // adopted set: it was produced on stream_copy itself, stream order covers it
    mark(c, 1);

    if (c->global_time == 0) {                                                           // .cpp:481-557
        M3 Rcam = c->rmats.back(); V3 tcam = c->tvecs.back();
        M3 Rcam_inv = m3_inverse(Rcam);
        int emptyVoxel[3] = {0, 0, 0};
        mark(c, 2); mark(c, 3);
        if ((r = do_integrate(c, Rcam_inv, tcam, emptyVoxel))) return r;
        mark(c, 4);
        TransformLevel tl[LEVELS];
        for (int i = 0; i < LEVELS; ++i) { tl[i].vs = c->vmaps_curr[i]; tl[i].ns = c->nmaps_curr[i]; tl[i].vd = c->vmaps_g_prev[i]; tl[i].nd = c->nmaps_g_prev[i]; tl[i].rows = rows >> i; tl[i].cols = cols >> i; }
        if ((r = transform_maps_pyramid(tl, LEVELS, to_mat33(Rcam.m), make_float3(tcam.v[0], tcam.v[1], tcam.v[2]), c->stream))) return r;
        mark(c, 5);
        ++c->global_time;
        c->current_utime = utime;
        record_dense_pose(c, true);                                                      // .cpp:529-536 (no outputPose on the first frame)
        if (out) kt_get_pose(c, out);
        return 0;
    }

    M3 Rprev = c->rmats.back(); V3 tprev = c->tvecs.back();
    M3 Rcurr = Rprev; V3 tcurr = tprev;
    if ((r = run_odometry(c, Rprev, tprev, &Rcurr, &tcurr))) return r;
    mark(c, 2);
    c->current_utime = utime;
    // rmats_.push_back / tvecs_.push_back (.cpp:578-579): only .back() is ever read (by the reference too), so the history is one entry deep --
    // the full trajectory is the dense pose graph (kt_get_dense_pose)
    c->rmats.back() = Rcurr; c->tvecs.back() = tcurr;

    for (int i = 0; i < 3; ++i) c->currentGlobalCamera[i] = global_camera(c->volumeBasis[i], c->size, c->voxelWrap[i], c->voxel, tcurr.v[i]);   // .cpp:581-596
    M3 Rcurr_inv = m3_inverse(Rcurr);                                                    // .cpp:627
    float currentTranslation[3];
    for (int i = 0; i < 3; ++i) currentTranslation[i] = c->tvecs.back().v[i] - c->volumeBasis[i];
    const int thresh = c->parked ? INT_MAX : c->cfg.voxel_shift;                         // .cpp:636
    int trans[3];
    shift_steps(currentTranslation, c->voxel, thresh, trans);                            // .cpp:642-667
    int vWrapCopy[3];
    for (int axis = 0; axis < 3; ++axis) {                                               // x :675-723, y :729-777, z :783-831
        vwrap_copy(c, vWrapCopy);
        const int n = trans[axis];
        int lo[3], hi[3];
        const int dir = shift_box(axis, n, thresh, c->overlap, V, lo, hi);              // kt_shift.hpp: which slab leaves the volume
        const bool cycled = dir != 0;
        if (cycled) {
            if ((r = fetch_cloud(c, vWrapCopy, lo, hi))) return r;
            if (c->slice_meshing && (r = mesh_box(c, vWrapCopy, lo, hi))) return r;
            if ((r = mg_barrier(c))) return r;                          // peers may still read my boundary plane for their extraction
            if ((r = clear_volume_shared(axis, dir < 0 ? 1 : 0, c->vv, V, c->voxelWrap[axis], c->voxelWrap[axis] + n, c->stream))) return r;
        }
        if (cycled) {                                                                    // mutexOutCloudBuffer (.cpp:1156-1208)
            int vt[3] = {0, 0, 0}; vt[axis] = n;
            float voxelTransSize[3];
            for (int i = 0; i < 3; ++i) voxelTransSize[i] = c->voxel * vt[i];
            // the slice is recorded before tvecs_.back() / voxelWrap move, with the camera of this frame
            for (int i = 0; i < 3; ++i) c->tvecs.back().v[i] -= voxelTransSize[i];
            const int dim = slice_dimension(vt);
            if ((r = push_slice(c, dim))) return r;
            for (int i = 0; i < 3; ++i) c->voxelWrap[i] += vt[i];
            for (int i = 0; i < 3; ++i) tcurr.v[i] -= voxelTransSize[i];
            ++c->shifted_last;
        }
    }
    vwrap_copy(c, vWrapCopy);
    // shared volume: every rank has cleared the leaving planes of ITS TSDF replica before any peer's integration stores into it
    if (c->shifted_last && (r = mg_barrier(c))) return r;
    mark(c, 3);

    if (c->timing) cudaEventRecord(c->ev_krn[0], c->stream);
    if ((r = do_integrate(c, Rcurr_inv, tcurr, vWrapCopy))) return r;                    // .cpp:864-876
    if (c->timing) cudaEventRecord(c->ev_krn[1], c->stream);
    if ((r = mg_barrier(c))) return r;                                                   // every slab holds this frame before any ray reads it
    mark(c, 4);
    vwrap_copy(c, vWrapCopy);
    RaycastArgs ra;
    ra.k.fx = c->cfg.fx; ra.k.fy = c->cfg.fy; ra.k.cx = c->cfg.cx; ra.k.cy = c->cfg.cy;
    ra.R = to_mat33(Rcurr.m); ra.t = make_float3(tcurr.v[0], tcurr.v[1], tcurr.v[2]); ra.trunc = c->trunc;
    ra.volume_size = make_float3(c->size, c->size, c->size); ra.tsdf = c->tsdf; ra.color = c->color; ra.vol = V;
    ra.wrap = make_int3(vWrapCopy[0], vWrapCopy[1], vWrapCopy[2]);
    for (int l = 0; l < LEVELS; ++l) { ra.vmap[l] = c->vmaps_g_prev[l]; ra.nmap[l] = c->nmaps_g_prev[l]; }
    ra.rows = rows; ra.cols = cols; ra.vmap_color = c->vmap_curr_color;
    ra.n_levels = (mode == 0 || mode == 2) ? LEVELS : 1;                                 // .cpp:892-899
    ra.multi = c->world > 1 ? 1 : 0;
    if (ra.multi) {
        ra.n_levels = LEVELS;
        ra.vv = c->vv;
        const int tiles_y = rows / 8;
        ra.tile_row_begin = c->rank * tiles_y / c->world; ra.tile_row_end = (c->rank + 1) * tiles_y / c->world;
        for (int g = 0; g < c->world; ++g) {
            for (int l = 0; l < LEVELS; ++l) { ra.peer_vmap[g][l] = (float*)(c->peer_arena[g] + c->off_vmap[l]); ra.peer_nmap[g][l] = (float*)(c->peer_arena[g] + c->off_nmap[l]); }
            ra.peer_vcol[g] = c->peer_arena[g] + c->off_vcol;
        }
    }
    if (c->timing) cudaEventRecord(c->ev_krn[2], c->stream);
    if ((r = raycast(ra, c->stream))) return r;
    if (c->timing) cudaEventRecord(c->ev_krn[3], c->stream);
    if ((r = mg_barrier(c))) return r;                                                   // all tiles of the predicted surface have landed everywhere
    mark(c, 5);
    // a cross-GPU barrier that timed out writes its flag straight into mapped host memory: report it with the frame it belongs to when it
    // has already fired (free to check), else with the next frame's pose read-back (run_odometry)
    if (c->world > 1 && *(volatile int*)c->mg_error_host) { set_error("cross-GPU barrier timed out waiting for rank %d", *c->mg_error_host - 1); return KT_ERR_STATE; }
    ++c->global_time;
    record_dense_pose(c, false);                                                         // .cpp:901-914
    if (out) kt_get_pose(c, out);
    return 0;
}

} // namespace

// ---------------------------------------------------------------------------------------------------
extern "C" {

const char* kt_last_error(void) { return kt::last_error(); }

int kt_cuda_available(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n > 0 ? 1 : 0;
}

int kt_reset(kt_ctx* c)
{
    if (!c) return KT_ERR_INVALID;
    c->global_time = 0;
    c->rmats.clear(); c->tvecs.clear();
    c->rmats.push_back(m3_identity());
    V3 tb = {{c->volumeBasis[0], c->volumeBasis[1], c->volumeBasis[2]}};
    c->tvecs.push_back(tb);
    for (int i = 0; i < 3; ++i) { c->voxelWrap[i] = 0; c->currentGlobalCamera[i] = c->volumeBasis[i] - c->size * 0.5f; }
    drop_slices(c);
    c->deformed.clear();
    if (c->deform_arena) c->deform_arena->rewind();
    c->loops.clear(); c->pgo_nodes.clear();
    c->dense_poses.clear();                      // reset(): densePoseGraph.clear(), latestDensePoseId = 0 (.cpp:300-301)
    c->trace_iters = 0; c->shifted_last = 0; c->cloud_count = 0;
    c->pf_valid = false; c->pf_built = false; c->frontend_ready = false; c->maps_on_stream = false;
    if (c->stream_copy) cudaStreamSynchronize(c->stream_copy);
    if (c->mg_error_host) { KT_CUDA(cudaStreamSynchronize(c->stream)); *c->mg_error_host = 0; }      // a timed-out cross-GPU barrier is not sticky across resets
    int r = init_shared(c->vv, c->cfg.vol, c->stream);
    if (r) return r;
    // Q7: stale y/z planes of invalid pixels start from a defined state (zeros)
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    for (int l = 0; l < LEVELS; ++l) {
        size_t Pl = P >> (2 * l);
        KT_CUDA(cudaMemsetAsync(c->vmaps_g_prev[l], 0, Pl * 12, c->stream)); KT_CUDA(cudaMemsetAsync(c->nmaps_g_prev[l], 0, Pl * 12, c->stream));
        KT_CUDA(cudaMemsetAsync(c->vmaps_curr[l], 0, Pl * 12, c->stream)); KT_CUDA(cudaMemsetAsync(c->nmaps_curr[l], 0, Pl * 12, c->stream));
        KT_CUDA(cudaMemsetAsync(c->vmaps_alt[l], 0, Pl * 12, c->stream)); KT_CUDA(cudaMemsetAsync(c->nmaps_alt[l], 0, Pl * 12, c->stream));
    }
    KT_CUDA(cudaMemsetAsync(c->vmap_curr_color, 0, P * 4, c->stream));
    KT_CUDA(cudaMemsetAsync(c->state, 0, sizeof(OdomState), c->stream));
    KT_CUDA(cudaStreamSynchronize(c->stream));
    return KT_OK;
}

int kt_create(const kt_config* cfg, kt_ctx** out)
{
    if (!cfg || !out) { set_error("kt_create: null argument"); return KT_ERR_INVALID; }
    if (cfg->rows <= 0 || cfg->cols <= 0 || cfg->vol < 32 || cfg->vol % 32 != 0 || cfg->volume_size <= 0) { set_error("kt_create: bad geometry (vol must be a multiple of 32)"); return KT_ERR_INVALID; }
    if ((cfg->rows % 8) != 0 || (cfg->cols % 32) != 0) { set_error("kt_create: rows must be a multiple of 8 and cols of 32"); return KT_ERR_INVALID; }
    if (cfg->odometry < 0 || cfg->odometry > 2) { set_error("kt_create: odometry must be 0, 1 or 2"); return KT_ERR_INVALID; }
    if (cfg->world > 1) {
        const int w = cfg->world;
        if (w > MAX_GPUS || (w & (w - 1)) || cfg->rank < 0 || cfg->rank >= w || (cfg->vol & (cfg->vol - 1)) || cfg->vol / w < 2) {
            set_error("kt_create: a shared volume needs world in {2,4,8}, 0 <= rank < world and a power-of-two vol"); return KT_ERR_INVALID; }
    }
    if (!kt_cuda_available()) { set_error("kt_create: no CUDA device (this library has no CPU path)"); return KT_ERR_CUDA; }
    KT_CUDA(cudaSetDevice(cfg->device));
    kt_ctx* c = new kt_ctx();
    c->cfg = *cfg;
    c->launches_at_create = g_launches.load();
    if (c->cfg.cloud_capacity <= 0) c->cfg.cloud_capacity = 3 * cfg->rows * cfg->cols;          // KintinuousTracker.cpp:77
    c->overlap = cfg->overlap; c->parked = cfg->parked;
    c->size = cfg->volume_size;
    c->voxel = c->size / (float)cfg->vol;
    c->trunc = trunc_dist_for(c->size, c->voxel);                                               // KintinuousTracker.cpp:112, TSDFVolume.cpp:96
    for (int i = 0; i < 3; ++i) c->volumeBasis[i] = c->size * 0.5f;                             // KintinuousTracker.cpp:109
    c->timing = false;
    {   // iteration schedules: ICPOdometry.cpp:42-55, RGBDOdometry.cpp:76-107
        const int icp[4] = {10, 5, 4, 0}, icpf[4] = {0, 10, 5, 0}, rgb[4] = {10, 7, 7, 7}, rgbf[4] = {0, 10, 7, 0}, ri[4] = {10, 5, 4, 0}, rif[4] = {0, 10, 7, 0};
        const int* sel = cfg->odometry == 0 ? (cfg->fast_odometry ? icpf : icp) : cfg->odometry == 1 ? (cfg->fast_odometry ? rgbf : rgb) : (cfg->fast_odometry ? rif : ri);
        for (int i = 0; i < 4; ++i) c->iterations[i] = sel[i];
    }
    int r = 0;
#define KT_TRY(x) do { r = (x); if (r) { kt_destroy(c); return r; } } while (0)
    r = kt::cuda_check(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking), "stream", __FILE__, __LINE__);
    if (r) { delete c; return r; }
    KT_TRY(kt::cuda_check(cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking), "stream2", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaEventCreateWithFlags(&c->ev_input, cudaEventDisableTiming), "event", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaEventCreateWithFlags(&c->ev_scaled, cudaEventDisableTiming), "event", __FILE__, __LINE__));
    const size_t P = (size_t)cfg->rows * cfg->cols;
    {   // shared arena: local volume slab, model maps, raycast colour, barrier flags -- one allocation, one IPC handle
        c->world = cfg->world > 1 ? cfg->world : 1; c->rank = cfg->world > 1 ? cfg->rank : 0;
        c->local_planes = cfg->vol / c->world;
        // colour planes are dealt to the ranks in blocks of mg_block storage planes (KT_MG_BLOCK, default max(8, V / 64)): small enough
        // that any viewing frustum spreads evenly over the ranks (the frustum's cross-section grows with depth: with V / 16-plane blocks
        // the farthest block alone would hold a third of the work), large enough to amortise the per-column set-up of integrate_kernel,
        // which walks one ownership block per CTA
        c->mg_block = cfg->vol / 64 > 8 ? cfg->vol / 64 : 8;
        { int b = 1; while (b * 2 <= c->mg_block) b *= 2; c->mg_block = b; }
        if (const char* e = getenv("KT_MG_BLOCK")) { int b = atoi(e); if (b >= 1 && (b & (b - 1)) == 0) c->mg_block = b; }
        while (c->mg_block > 1 && c->mg_block * c->world > cfg->vol) c->mg_block >>= 1;
        if (c->world == 1) c->mg_block = 1;
        auto al = [](size_t x) { return (x + 255) / 256 * 256; };
        size_t off = 0;
        const size_t plane_vox = (size_t)cfg->vol * cfg->vol;
        c->off_tsdf = off; off = al(off + plane_vox * cfg->vol * 2);                   // full replica
        c->off_color = off; off = al(off + plane_vox * c->local_planes * 4);            // this rank's planes
        for (int l = 0; l < LEVELS; ++l) { size_t Pl = P >> (2 * l); c->off_vmap[l] = off; off = al(off + Pl * 12); c->off_nmap[l] = off; off = al(off + Pl * 12); }
        c->off_vcol = off; off = al(off + P * 4);
        c->off_flags = off; off = al(off + 256);
        c->off_xwords = off; off = al(off + odom_exchange_words() * sizeof(unsigned long long));      // in the arena so that peers can add to them
        c->arena_bytes = off;
        KT_TRY(dev_alloc(c, &c->arena, off));
        KT_TRY(kt::cuda_check(cudaMemset(c->arena + c->off_flags, 0, 256), "memset", __FILE__, __LINE__));
        c->xwords_dev = (unsigned long long*)(c->arena + c->off_xwords);
        KT_TRY(kt::cuda_check(cudaMemset(c->xwords_dev, 0, odom_exchange_words() * sizeof(unsigned long long)), "memset", __FILE__, __LINE__)); c->xwords_clean = true;
        c->split_icp = c->world > 1 && getenv("KT_MG_SPLIT_ICP") != nullptr;
        c->tsdf = (int16_t*)(c->arena + c->off_tsdf); c->color = c->arena + c->off_color;
        for (int g = 0; g < MAX_GPUS; ++g) c->peer_arena[g] = c->arena;
        c->connected = (c->world == 1);
        c->epoch = 0;
        c->vv = single_volume(c->tsdf, c->color, cfg->vol);
        c->vv.world = c->world; c->vv.rank = c->rank;
        c->vv.bshift = 0; { int t = c->mg_block; while (t > 1) { t >>= 1; ++c->vv.bshift; } }
        c->vv.nshift = 0; { int t = c->world; while (t > 1) { t >>= 1; ++c->vv.nshift; } }
        KT_TRY(dev_alloc(c, &c->peer_flags_dev, (size_t)MAX_GPUS)); 
        // the barrier's time-out flag lives in MAPPED host memory: the kernel writes it in place, the host reads it with the pose (no copy)
        KT_TRY(kt::cuda_check(cudaHostAlloc((void**)&c->mg_error_host, sizeof(int), cudaHostAllocMapped), "mapped", __FILE__, __LINE__)); *c->mg_error_host = 0;
        KT_TRY(kt::cuda_check(cudaHostGetDevicePointer((void**)&c->mg_error_dev, c->mg_error_host, 0), "mapped alias", __FILE__, __LINE__));
    }
    KT_TRY(dev_alloc(c, &c->depth_raw, P)); KT_TRY(dev_alloc(c, &c->rgb, P * 3));
    KT_TRY(dev_alloc(c, &c->depth_alt, P)); KT_TRY(dev_alloc(c, &c->rgb_alt, P * 3)); c->pf_valid = false; c->pf_depth = c->pf_rgb = 0;
    KT_TRY(kt::cuda_check(cudaStreamCreateWithFlags(&c->stream_copy, cudaStreamNonBlocking), "stream_copy", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaEventCreateWithFlags(&c->ev_prefetch, cudaEventDisableTiming), "event", __FILE__, __LINE__));
    for (int i = 0; i < 2; ++i) KT_TRY(kt::cuda_check(cudaEventCreateWithFlags(&c->ev_done[i], cudaEventDisableTiming), "event", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaEventCreateWithFlags(&c->ev_maps, cudaEventDisableTiming), "event", __FILE__, __LINE__)); c->maps_on_stream = false;
    c->last_parity = 0;
    for (int l = 0; l < LEVELS; ++l) {
        size_t Pl = P >> (2 * l);
        KT_TRY(dev_alloc(c, &c->depths_curr[l], Pl));
        c->vmaps_g_prev[l] = (float*)(c->arena + c->off_vmap[l]); c->nmaps_g_prev[l] = (float*)(c->arena + c->off_nmap[l]);
        KT_TRY(dev_alloc(c, &c->vmaps_curr[l], Pl * 3)); KT_TRY(dev_alloc(c, &c->nmaps_curr[l], Pl * 3));
        KT_TRY(dev_alloc(c, &c->depths_alt[l], Pl)); KT_TRY(dev_alloc(c, &c->vmaps_alt[l], Pl * 3)); KT_TRY(dev_alloc(c, &c->nmaps_alt[l], Pl * 3));
        c->lastDepth[l] = c->nextDepth[l] = 0; c->lastImage[l] = c->nextImage[l] = 0; c->nextdIdx[l] = c->nextdIdy[l] = 0; c->pointClouds[l] = 0; c->corresImg[l] = 0;
        if (cfg->odometry != 0) {
            KT_TRY(dev_alloc(c, &c->lastDepth[l], Pl)); KT_TRY(dev_alloc(c, &c->nextDepth[l], Pl));
            KT_TRY(dev_alloc(c, &c->lastImage[l], Pl)); KT_TRY(dev_alloc(c, &c->nextImage[l], Pl));
            KT_TRY(dev_alloc(c, &c->nextdIdx[l], Pl)); KT_TRY(dev_alloc(c, &c->nextdIdy[l], Pl));
            KT_TRY(dev_alloc(c, &c->pointClouds[l], Pl * 3));
            uint8_t* ci = 0; KT_TRY(dev_alloc(c, &ci, Pl * 16)); c->corresImg[l] = ci;
        }
    }
    c->vmap_curr_color = c->arena + c->off_vcol; KT_TRY(dev_alloc(c, &c->depth_scaled, P)); KT_TRY(dev_alloc(c, &c->depth_scaled_alt, P)); c->pf_built = false; c->frontend_ready = false;
    KT_TRY(dev_alloc(c, &c->ztable, (size_t)2 * cfg->vol)); KT_TRY(dev_alloc(c, &c->cw_scratch, P)); KT_TRY(dev_alloc(c, &c->rgbf_scratch, P * 4)); KT_TRY(dev_alloc(c, &c->cw_alt, P)); KT_TRY(dev_alloc(c, &c->rgbf_alt, P * 4));

    KT_TRY(dev_alloc(c, &c->state, 1)); KT_TRY(dev_alloc(c, &c->partials, (size_t)MAX_PARTIALS * 32));
    KT_TRY(kt::cuda_check(cudaMemset(c->partials, 0, (size_t)MAX_PARTIALS * 32 * sizeof(float)), "memset", __FILE__, __LINE__));   // tags start at 0
    KT_TRY(dev_alloc(c, &c->bar_dev, 1)); KT_TRY(kt::cuda_check(cudaMemset(c->bar_dev, 0, sizeof(unsigned int)), "memset", __FILE__, __LINE__)); c->bar_count = 0;
    KT_TRY(dev_alloc(c, &c->prof_dev, 64 * 8)); KT_TRY(dev_alloc(c, &c->ipartials, (size_t)MAX_PARTIALS * 2));
    KT_TRY(dev_alloc(c, &c->trace_dev, (size_t)MAX_TRACE_ITERS * TRACE_STRIDE)); KT_TRY(dev_alloc(c, &c->pose12_dev, 12));
    c->cloud_capacity = (size_t)c->cfg.cloud_capacity;
    KT_TRY(dev_alloc(c, &c->cloud_dev, c->cloud_capacity)); KT_TRY(dev_alloc(c, &c->counter_dev, 1));
    c->slice_arena = new PinnedArena();
    c->mesh_weight_cull = 8;                                   // -cw default, also the live mesh's until kt_set_slice_meshing
    if (!c->slice_arena->alloc(256)) { set_error("kt_create: pinned slice arena"); kt_destroy(c); return KT_ERR_CUDA; }      // the first 64 MB slab now, not inside the first shift frame
    c->slice_arena->rewind();
    KT_TRY(kt::cuda_check(cudaStreamCreateWithFlags(&c->stream_slices, cudaStreamNonBlocking), "stream_slices", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaEventCreateWithFlags(&c->ev_cloud_ready, cudaEventDisableTiming), "event", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaEventCreateWithFlags(&c->ev_cloud_free, cudaEventDisableTiming), "event", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaMallocHost((void**)&c->pose12_host, 12 * sizeof(float)), "pinned", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaHostAlloc((void**)&c->result_host, sizeof(OdomResult), cudaHostAllocMapped), "pinned", __FILE__, __LINE__));
    std::memset(c->result_host, 0, sizeof(OdomResult));
    { void* dp = 0; KT_TRY(kt::cuda_check(cudaHostGetDevicePointer(&dp, c->result_host, 0), "mapped", __FILE__, __LINE__)); c->result_dev_alias = (float*)dp; }
    c->pose_seq = 0; c->pose_spin = getenv("KT_NO_POSE_SPIN") == nullptr;
    KT_TRY(kt::cuda_check(cudaMallocHost((void**)&c->trace_host, (size_t)MAX_TRACE_ITERS * TRACE_STRIDE * sizeof(float)), "pinned", __FILE__, __LINE__));
    KT_TRY(kt::cuda_check(cudaMallocHost((void**)&c->counter_host, sizeof(unsigned int)), "pinned", __FILE__, __LINE__));
    for (int i = 0; i < 7; ++i) KT_TRY(kt::cuda_check(cudaEventCreate(&c->ev[i]), "event", __FILE__, __LINE__));
    for (int i = 0; i < 2; ++i) KT_TRY(kt::cuda_check(cudaEventCreate(&c->ev_icp[i]), "event", __FILE__, __LINE__));
    for (int i = 0; i < 4; ++i) KT_TRY(kt::cuda_check(cudaEventCreate(&c->ev_krn[i]), "event", __FILE__, __LINE__));
    for (int i = 0; i < 2; ++i) KT_TRY(kt::cuda_check(cudaEventCreate(&c->ev_span[i]), "event", __FILE__, __LINE__));
    for (int i = 0; i < 6; ++i) c->stage_ms[i] = 0.f;
    KT_TRY(kt_reset(c));
#undef KT_TRY
    *out = c;
    return KT_OK;
}

int kt_destroy(kt_ctx* c)
{
    if (!c) return KT_OK;
    cudaSetDevice(c->cfg.device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    for (int g = 0; g < MAX_GPUS; ++g) if (c->peer_arena[g] && c->peer_arena[g] != c->arena) cudaIpcCloseMemHandle(c->peer_arena[g]);
    if (c->mg_error_host) cudaFreeHost(c->mg_error_host);
    drop_slices(c);
    if (c->pose_log) fclose(c->pose_log);
    if (c->slice_arena) { c->slice_arena->release(); delete c->slice_arena; }
    if (c->deform_arena) { c->deform_arena->release(); delete c->deform_arena; }
    slice_ws_free(&c->slice_ws);
    mesh_ws_free(&c->mesh_ws);
    if (c->mesh_verts_dev) cudaFree(c->mesh_verts_dev);
    if (c->mesh_tris_dev) cudaFree(c->mesh_tris_dev);
    if (c->stream_slices) cudaStreamDestroy(c->stream_slices);
    if (c->ev_cloud_ready) cudaEventDestroy(c->ev_cloud_ready);
    if (c->ev_cloud_free) cudaEventDestroy(c->ev_cloud_free);
    for (void* p : c->allocs) cudaFree(p);
    if (c->pose12_host) cudaFreeHost(c->pose12_host);
    if (c->result_host) cudaFreeHost(c->result_host);
    if (c->trace_host) cudaFreeHost(c->trace_host);
    if (c->counter_host) cudaFreeHost(c->counter_host);
    for (int i = 0; i < 7; ++i) if (c->ev[i]) cudaEventDestroy(c->ev[i]);
    for (int i = 0; i < 2; ++i) if (c->ev_icp[i]) cudaEventDestroy(c->ev_icp[i]);
    for (int i = 0; i < 4; ++i) if (c->ev_krn[i]) cudaEventDestroy(c->ev_krn[i]);
    for (int i = 0; i < 2; ++i) if (c->ev_span[i]) cudaEventDestroy(c->ev_span[i]);
    if (c->stream2) { cudaStreamSynchronize(c->stream2); cudaStreamDestroy(c->stream2); }
    if (c->stream_copy) { cudaStreamSynchronize(c->stream_copy); cudaStreamDestroy(c->stream_copy); }
    if (c->ev_prefetch) cudaEventDestroy(c->ev_prefetch);
    if (c->ev_maps) cudaEventDestroy(c->ev_maps);
    for (int i = 0; i < 2; ++i) if (c->ev_done[i]) cudaEventDestroy(c->ev_done[i]);
    if (c->ev_input) cudaEventDestroy(c->ev_input);
    if (c->ev_scaled) cudaEventDestroy(c->ev_scaled);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
    return KT_OK;
}

// If (depth, rgb) is the frame kt_prefetch_frame was given, make the prefetched buffer set the current one.
static bool adopt_prefetched(kt_ctx* c, const void* depth, const void* rgb)
{
    if (!(c->pf_valid && c->pf_depth == depth && c->pf_rgb == rgb)) {
        // a stale hint is dropped; its front end may still be writing the photometric "next" buffers this frame is about to rebuild
        if (c->pf_valid) cudaStreamWaitEvent(c->stream, c->ev_prefetch, 0);
        c->pf_valid = false; c->pf_built = false;
        return false;
    }
    std::swap(c->depth_raw, c->depth_alt); std::swap(c->rgb, c->rgb_alt);
    if (c->pf_built) {
        std::swap(c->depth_scaled, c->depth_scaled_alt); std::swap(c->cw_scratch, c->cw_alt); std::swap(c->rgbf_scratch, c->rgbf_alt);
        for (int l = 0; l < LEVELS; ++l) { std::swap(c->depths_curr[l], c->depths_alt[l]); std::swap(c->vmaps_curr[l], c->vmaps_alt[l]); std::swap(c->nmaps_curr[l], c->nmaps_alt[l]); }
        c->frontend_ready = true;
    }
    cudaStreamWaitEvent(c->stream, c->ev_prefetch, 0);          // the compute stream waits for the copy (and the front end)
    c->pf_valid = false; c->pf_built = false;
    return true;
}

static int finish_frame(kt_ctx* c, int r)
{
    c->frontend_ready = false;
    c->last_parity ^= 1;
    cudaEventRecord(c->ev_done[c->last_parity], c->stream);      // completion of this frame's last kernel
    return r;
}

int kt_process_frame_device(kt_ctx* c, const uint16_t* depth_dev, const uint8_t* rgb_dev, uint64_t utime, kt_pose* out)
{
    if (!c || !depth_dev || !rgb_dev) { set_error("kt_process_frame_device: null argument"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    if (!adopt_prefetched(c, depth_dev, rgb_dev)) {
        KT_CUDA(cudaMemcpyAsync(c->depth_raw, depth_dev, P * 2, cudaMemcpyDeviceToDevice, c->stream));
        KT_CUDA(cudaMemcpyAsync(c->rgb, rgb_dev, P * 3, cudaMemcpyDeviceToDevice, c->stream));
    }
    return finish_frame(c, process_frame_device(c, utime, out));
}

int kt_process_frame(kt_ctx* c, const uint16_t* depth_host, const uint8_t* rgb_host, uint64_t utime, kt_pose* out)
{
    if (!c || !depth_host || !rgb_host) { set_error("kt_process_frame: null argument"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    if (!adopt_prefetched(c, depth_host, rgb_host)) {
        KT_CUDA(cudaMemcpyAsync(c->depth_raw, depth_host, P * 2, cudaMemcpyHostToDevice, c->stream));   // TrackerInterface.cpp:90
        KT_CUDA(cudaMemcpyAsync(c->rgb, rgb_host, P * 3, cudaMemcpyHostToDevice, c->stream));           // TrackerInterface.cpp:91
    }
    return finish_frame(c, process_frame_device(c, utime, out));
}

int kt_prefetch_frame(kt_ctx* c, const uint16_t* depth, const uint8_t* rgb)
{
    if (!c || !depth || !rgb) { set_error("kt_prefetch_frame: null argument"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    // the spare set was last read by the frame BEFORE the last one; wait for that frame's completion event only, so the copy and the
    // front end overlap the last frame's integrate / ray-cast.  Host (pinned) or device pointers.
    KT_CUDA(cudaStreamWaitEvent(c->stream_copy, c->ev_done[c->last_parity ^ 1], 0));
    KT_CUDA(cudaMemcpyAsync(c->depth_alt, depth, P * 2, cudaMemcpyDefault, c->stream_copy));
    KT_CUDA(cudaMemcpyAsync(c->rgb_alt, rgb, P * 3, cudaMemcpyDefault, c->stream_copy));
    c->pf_built = false;
    static const bool lookahead = getenv("KT_NO_LOOKAHEAD") == nullptr;       // A/B knob: copy only
    if (lookahead && c->global_time > 0) {
        // invalid pixels keep the y/z planes of the previous frame's maps = the set that is current now (Q7); if that set was built on the
        // compute stream (frame not prefetched, e.g. frame 0), wait for its front end -- not for the whole frame
        if (c->maps_on_stream) KT_CUDA(cudaStreamWaitEvent(c->stream_copy, c->ev_maps, 0));
        // photometric odometry: its "next" pyramids were swapped to "last" when the previous frame's odometry finished, so the
        // buffers now called next are free until the coming frame
        const bool ph = c->cfg.odometry != 0;
        int r = build_frontend(c, c->depth_alt, c->rgb_alt, c->depth_scaled_alt, c->depths_alt, c->vmaps_alt, c->nmaps_alt, c->vmaps_curr, c->nmaps_curr,
                               c->cw_alt, c->rgbf_alt, ph ? c->nextDepth : 0, ph ? c->nextImage : 0, c->stream_copy);
        if (r) return r;
        c->pf_built = true;
    }
    KT_CUDA(cudaEventRecord(c->ev_prefetch, c->stream_copy));
    c->pf_depth = depth; c->pf_rgb = rgb; c->pf_valid = true;
    return KT_OK;
}

int kt_finalise(kt_ctx* c)                                                                           // KintinuousTracker::finalise (.cpp:1003-1048)
{
    if (!c) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    int vWrapCopy[3]; vwrap_copy(c, vWrapCopy);
    const int V = c->cfg.vol;
    int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
    int r = fetch_cloud(c, vWrapCopy, lo, hi);
    if (r) return r;
    if (c->slice_meshing && (r = mesh_box(c, vWrapCopy, lo, hi))) return r;
    return push_slice(c, 7);     // CloudSlice::FINAL
}

int kt_get_pose(kt_ctx* c, kt_pose* out)
{
    if (!c || !out) return KT_ERR_INVALID;
    for (int i = 0; i < 9; ++i) out->R[i] = c->rmats.back().m[i];
    for (int i = 0; i < 3; ++i) { out->t[i] = c->tvecs.back().v[i]; out->global_t[i] = c->currentGlobalCamera[i]; out->voxel_wrap[i] = c->voxelWrap[i]; }
    out->shifted = c->shifted_last;
    out->frame = c->global_time;
    return KT_OK;
}

float kt_get_voxel_size(kt_ctx* c) { return c ? c->voxel : 0.f; }
float kt_get_trunc_dist(kt_ctx* c) { return c ? c->trunc : 0.f; }
int kt_set_overlap(kt_ctx* c, int overlap) { if (!c) return KT_ERR_INVALID; c->overlap = overlap; return KT_OK; }
int kt_set_parked(kt_ctx* c, int parked) { if (!c) return KT_ERR_INVALID; c->parked = parked; return KT_OK; }
int kt_num_slices(kt_ctx* c) { return c ? (int)c->slices.size() : 0; }

int kt_get_slice(kt_ctx* c, int idx, kt_point_xyzrgb* points, size_t max_points, size_t* count, int* dimension, float* camera_t)
{
    if (!c || idx < 0 || idx >= (int)c->slices.size()) { set_error("kt_get_slice: bad index"); return KT_ERR_INVALID; }
    const SliceRec& s = c->slices[idx];
    if (count) *count = s.count;
    if (dimension) *dimension = s.dimension;
    if (camera_t) for (int i = 0; i < 3; ++i) camera_t[i] = s.camera_t[i];
    size_t n = std::min(max_points, s.count);
    if (points && n) {
        KT_CUDA(cudaEventSynchronize(s.ready));                  // the asynchronous download of this slice has landed
        std::memcpy(points, s.points, n * sizeof(kt_point_xyzrgb));
    }
    return KT_OK;
}

int kt_num_dense_poses(kt_ctx* c) { return c ? (int)c->dense_poses.size() : 0; }
int kt_get_dense_pose(kt_ctx* c, int idx, kt_dense_pose* out)
{
    if (!c || !out || idx < 0 || idx >= (int)c->dense_poses.size()) { set_error("kt_get_dense_pose: bad argument"); return KT_ERR_INVALID; }
    *out = c->dense_poses[idx];
    return KT_OK;
}
int kt_set_pose_log(kt_ctx* c, const char* path)
{
    if (!c) return KT_ERR_INVALID;
    if (c->pose_log) { fclose(c->pose_log); c->pose_log = 0; }
    if (path && *path) {
        c->pose_log = fopen(path, "a");                       // std::fstream::app (.cpp:205)
        if (!c->pose_log) { set_error("kt_set_pose_log: cannot open %s", path); return KT_ERR_INVALID; }
    }
    return KT_OK;
}
int kt_format_pose_line(uint64_t timestamp, const float* global_t3, const float* R9, char* buf, size_t capacity)
{
    if (!global_t3 || !R9 || !buf) return KT_ERR_INVALID;
    return format_pose_line(timestamp, global_t3, R9, buf, capacity) < 0 ? KT_ERR_CAPACITY : KT_OK;
}

int kt_set_slice_processing(kt_ctx* c, int enabled, int weight_cull)
{
    if (!c) return KT_ERR_INVALID;
    c->slice_processing = enabled != 0; c->slice_weight_cull = weight_cull;
    return KT_OK;
}

int kt_get_processed_slice(kt_ctx* c, int idx, kt_point_xyzrgbnormal* points, size_t max_points, size_t* count)
{
    if (!c || idx < 0 || idx >= (int)c->slices.size()) { set_error("kt_get_processed_slice: bad index"); return KT_ERR_INVALID; }
    const SliceRec& s = c->slices[idx];
    if (!s.has_processed) { set_error("kt_get_processed_slice: slice %d was recorded with slice processing off (kt_set_slice_processing)", idx); return KT_ERR_STATE; }
    if (count) *count = s.processed_count;
    size_t n = std::min(max_points, s.processed_count);
    if (points && n) {
        KT_CUDA(cudaEventSynchronize(s.ready));
        std::memcpy(points, s.processed, n * sizeof(kt_point_xyzrgbnormal));
    }
    return KT_OK;
}

int kt_set_slice_meshing(kt_ctx* c, int enabled, int weight_cull)
{
    if (!c) return KT_ERR_INVALID;
    if (c->world > 1 && enabled) { set_error("kt_set_slice_meshing: a volume shared by %d GPUs cannot be meshed", c->world); return KT_ERR_INVALID; }
    c->slice_meshing = enabled != 0; c->mesh_weight_cull = weight_cull;
    return KT_OK;
}

int kt_get_slice_mesh(kt_ctx* c, int idx, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris, size_t* n_verts, size_t* n_tris)
{
    if (!c || idx < 0 || idx >= (int)c->slices.size()) { set_error("kt_get_slice_mesh: bad index"); return KT_ERR_INVALID; }
    const SliceRec& s = c->slices[idx];
    if (!s.has_mesh) { set_error("kt_get_slice_mesh: slice %d was recorded with meshing off (kt_set_slice_meshing)", idx); return KT_ERR_STATE; }
    if (n_verts) *n_verts = s.mesh_nv;
    if (n_tris) *n_tris = s.mesh_nt;
    const size_t nv = verts ? std::min(max_verts, s.mesh_nv) : 0, nt = tris ? std::min(max_tris, s.mesh_nt) : 0;
    if (nv || nt) KT_CUDA(cudaEventSynchronize(s.ready));
    if (nv) std::memcpy(verts, s.mesh_verts, nv * sizeof(kt_mesh_vertex));
    if (nt) std::memcpy(tris, s.mesh_tris, nt * 3 * sizeof(uint32_t));
    return KT_OK;
}

int kt_get_live_mesh(kt_ctx* c, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris, size_t* n_verts, size_t* n_tris)
{
    if (!c) return KT_ERR_INVALID;
    if (c->world > 1) { set_error("kt_get_live_mesh: a volume shared by %d GPUs cannot be meshed", c->world); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    int vWrapCopy[3]; vwrap_copy(c, vWrapCopy);
    const int V = c->cfg.vol;
    int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
    int r = mesh_box(c, vWrapCopy, lo, hi);
    if (r) return r;
    if (n_verts) *n_verts = c->mesh_nv;
    if (n_tris) *n_tris = c->mesh_nt;
    const size_t nv = verts ? std::min(max_verts, c->mesh_nv) : 0, nt = tris ? std::min(max_tris, c->mesh_nt) : 0;
    if (nv) KT_CUDA(cudaMemcpyAsync(verts, c->mesh_verts_dev, nv * sizeof(kt_mesh_vertex), cudaMemcpyDeviceToHost, c->stream));
    if (nt) KT_CUDA(cudaMemcpyAsync(tris, c->mesh_tris_dev, nt * 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(cudaStreamSynchronize(c->stream));
    return KT_OK;
}

// The meshes of the first n_slices slices as one binary PLY; with `deformed`, the vertices of the last kt_deform_map
static int save_mesh_ply(kt_ctx* c, const char* path, size_t n_slices, bool deformed, const char* who)
{
    size_t nv = 0, nt = 0; bool any = false;
    for (size_t i = 0; i < n_slices; ++i) { const auto& s = c->slices[i]; if (s.has_mesh) { any = true; nv += s.mesh_nv; nt += s.mesh_nt; } }
    if (!any) { set_error("%s: no slice was recorded with meshing on (kt_set_slice_meshing)", who); return KT_ERR_STATE; }
    if (nv > 0x7fffffffu) { set_error("%s: %zu vertices do not fit the PLY's int indices", who, nv); return KT_ERR_CAPACITY; }
    FILE* f = fopen(path, "wb");
    if (!f) { set_error("%s: cannot open %s", who, path); return KT_ERR_INVALID; }
    fprintf(f, "ply\nformat binary_little_endian 1.0\nelement vertex %zu\nproperty float x\nproperty float y\nproperty float z\n"
               "property float nx\nproperty float ny\nproperty float nz\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n"
               "element face %zu\nproperty list uchar int vertex_indices\nend_header\n", nv, nt);
    std::vector<unsigned char> buf;
    bool ok = true;
    for (size_t k = 0; k < n_slices; ++k) {                        // x86 / aarch64 hosts are little-endian: records are the raw bytes
        const auto& s = c->slices[k];
        if (!s.has_mesh || !s.mesh_nv) continue;
        if (cudaEventSynchronize(s.ready) != cudaSuccess) { ok = false; break; }
        const kt_mesh_vertex* mv = deformed ? c->deformed[k].mesh_verts : s.mesh_verts;
        buf.resize(s.mesh_nv * 27);
        for (size_t i = 0; i < s.mesh_nv; ++i) {
            std::memcpy(&buf[i * 27], &mv[i].x, 24);
            buf[i * 27 + 24] = mv[i].r; buf[i * 27 + 25] = mv[i].g; buf[i * 27 + 26] = mv[i].b;
        }
        ok = ok && fwrite(buf.data(), 1, buf.size(), f) == buf.size();
    }
    uint32_t base = 0;
    for (size_t k = 0; k < n_slices; ++k) {
        const auto& s = c->slices[k];
        if (!ok) break;
        if (!s.has_mesh) continue;
        buf.resize(s.mesh_nt * 13);
        for (size_t t = 0; t < s.mesh_nt; ++t) {
            buf[t * 13] = 3;
            for (int k = 0; k < 3; ++k) { const int32_t v = (int32_t)(s.mesh_tris[3 * t + k] + base); std::memcpy(&buf[t * 13 + 1 + 4 * k], &v, 4); }
        }
        ok = ok && fwrite(buf.data(), 1, buf.size(), f) == buf.size();
        base += (uint32_t)s.mesh_nv;
    }
    if (fclose(f) != 0) ok = false;
    if (!ok) { set_error("%s: writing %s failed", who, path); return KT_ERR_CUDA; }
    return KT_OK;
}

int kt_save_mesh_ply(kt_ctx* c, const char* path)
{
    if (!c || !path) return KT_ERR_INVALID;
    return save_mesh_ply(c, path, c->slices.size(), false, "kt_save_mesh_ply");
}

// The deformation graph's nodes (initialiseGraphPoses): the dense pose graph's positions, the first and every one more than node_spacing
// from the last taken.  KT_ERR_STATE without a recorded map, with fewer than k + 1 nodes or with descending timestamps.
static int deform_nodes(kt_ctx* c, float node_spacing, std::vector<float>& npos, std::vector<uint64_t>& ntime, const char* who)
{
    bool any = false;
    for (const auto& s : c->slices) if (s.has_processed || s.has_mesh) any = true;
    if (!any) { set_error("%s: no processed slice and no slice mesh recorded (kt_set_slice_processing / kt_set_slice_meshing)", who); return KT_ERR_STATE; }
    const size_t nd = c->dense_poses.size();
    std::vector<float> gpos(nd * 3);
    for (size_t i = 0; i < nd; ++i) for (int e = 0; e < 3; ++e) gpos[3 * i + e] = c->dense_poses[i].pose[4 * e + 3];
    const std::vector<int> take = deform_sample_nodes(gpos.data(), nd, node_spacing);
    const int nn = (int)take.size();
    if (nn < DEFORM_K + 1) {
        set_error("%s: node_spacing %g m leaves %d graph nodes on the trajectory; at least %d are needed", who, (double)node_spacing, nn, DEFORM_K + 1);
        return KT_ERR_STATE;
    }
    npos.resize(3 * (size_t)nn); ntime.resize(nn);
    for (int j = 0; j < nn; ++j) { ntime[j] = c->dense_poses[take[j]].timestamp; for (int e = 0; e < 3; ++e) npos[3 * j + e] = gpos[3 * take[j] + e]; }
    for (int j = 1; j < nn; ++j)
        if (ntime[j] < ntime[j - 1]) { set_error("%s: the dense pose graph's timestamps are not ascending", who); return KT_ERR_STATE; }
    return 0;
}

// Deformation::addCameraLoop's graph work (Deformation.cpp:264-318: appendVertices, the constraints, optimiseGraphSparse,
// applyGraphToVertices) over the map recorded so far, on the tracker's stream, with checked, finite constraints.  Nothing the tracker
// reads is written; c->deformed holds the result (cleared on an error).
static int deform_run(kt_ctx* c, const std::vector<float>& npos, const std::vector<uint64_t>& ntime, const std::vector<DeformConstraint>& cons,
                      kt_deform_report* report)
{
    const int nn = (int)ntime.size();
    size_t np = 0, nm = 0;
    for (const auto& s : c->slices) {
        if (s.has_processed) np += s.processed_count;
        if (s.has_mesh) nm += s.mesh_nv;
    }
    const size_t m = cons.size();
    std::vector<float> csrc(3 * m); std::vector<double> cdst(3 * m); std::vector<uint64_t> ct(m);
    for (size_t l = 0; l < m; ++l) { ct[l] = cons[l].time; for (int e = 0; e < 3; ++e) { csrc[3 * l + e] = cons[l].src[e]; cdst[3 * l + e] = cons[l].dst[e]; } }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    if (c->stream_slices) KT_CUDA(cudaStreamSynchronize(c->stream_slices));           // every slice has landed in its pinned buffers
    const size_t nmax = std::max(std::max(np, nm), m);
    float* d_npos = 0; uint64_t* d_ntime = 0; double* d_x = 0; uint64_t* d_t = 0; int32_t* d_ids = 0; double* d_w = 0; void* d_in = 0; void* d_out = 0;
    auto cleanup = [&]() { cudaFree(d_npos); cudaFree(d_ntime); cudaFree(d_x); cudaFree(d_t); cudaFree(d_ids); cudaFree(d_w); cudaFree(d_in); cudaFree(d_out); };
    auto run = [&]() -> int {
        cudaStream_t s = c->stream;
        KT_CUDA(cudaMalloc((void**)&d_npos, npos.size() * sizeof(float)));
        KT_CUDA(cudaMalloc((void**)&d_ntime, ntime.size() * sizeof(uint64_t)));
        KT_CUDA(cudaMalloc((void**)&d_x, (size_t)nn * 12 * sizeof(double)));
        KT_CUDA(cudaMalloc((void**)&d_t, nmax * sizeof(uint64_t)));
        KT_CUDA(cudaMalloc((void**)&d_ids, nmax * 4 * sizeof(int32_t)));
        KT_CUDA(cudaMalloc((void**)&d_w, nmax * 4 * sizeof(double)));
        KT_CUDA(cudaMalloc(&d_in, nmax * sizeof(kt_point_xyzrgbnormal)));
        KT_CUDA(cudaMemcpyAsync(d_npos, npos.data(), npos.size() * sizeof(float), cudaMemcpyHostToDevice, s));
        KT_CUDA(cudaMemcpyAsync(d_ntime, ntime.data(), ntime.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
        // constraint weights (their sources are vertices of the graph too: appendVertices) -> optimiseGraphSparse
        KT_CUDA(cudaMemcpyAsync(d_in, csrc.data(), csrc.size() * sizeof(float), cudaMemcpyHostToDevice, s));
        KT_CUDA(cudaMemcpyAsync(d_t, ct.data(), m * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
        int r = deform_weights(d_npos, d_ntime, nn, d_in, 2, d_t, m, d_ids, d_w, s); if (r) return r;
        std::vector<int32_t> cids(4 * m); std::vector<double> cw(4 * m);
        KT_CUDA(cudaMemcpyAsync(cids.data(), d_ids, cids.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        KT_CUDA(cudaMemcpyAsync(cw.data(), d_w, cw.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
        KT_CUDA(cudaStreamSynchronize(s));
        r = deform_optimise(npos.data(), nn, csrc.data(), cdst.data(), cids.data(), cw.data(), m, d_x, report, s); if (r) return r;
        c->deformed.assign(c->slices.size(), kt_ctx::Deformed());
        for (size_t i = 0; i < c->slices.size(); ++i) { c->deformed[i].processed = c->slices[i].processed; c->deformed[i].mesh_verts = c->slices[i].mesh_verts; }
        if (!report->deformed) return 0;                                                  // the map as recorded
        if (!c->deform_arena) c->deform_arena = new PinnedArena();
        c->deform_arena->rewind();
        KT_CUDA(cudaMalloc(&d_out, nmax * sizeof(kt_point_xyzrgbnormal)));
        // the map, one kind at a time: upload from the slices' pinned buffers, weights, apply, download into the deformation arena
        for (int kind = 0; kind < 2; ++kind) {
            const size_t total = kind == 0 ? np : nm, rec = kind == 0 ? sizeof(kt_point_xyzrgbnormal) : sizeof(kt_mesh_vertex);
            if (!total) continue;
            std::vector<uint64_t> vt(total);
            size_t off = 0;
            for (const auto& sl : c->slices) {
                const size_t cnt = kind == 0 ? (sl.has_processed ? sl.processed_count : 0) : (sl.has_mesh ? sl.mesh_nv : 0);
                if (!cnt) continue;
                KT_CUDA(cudaMemcpyAsync((char*)d_in + off * rec, kind == 0 ? (const void*)sl.processed : (const void*)sl.mesh_verts, cnt * rec, cudaMemcpyHostToDevice, s));
                std::fill(vt.begin() + off, vt.begin() + off + cnt, sl.utime);             // a vertex's time is its slice's
                off += cnt;
            }
            KT_CUDA(cudaMemcpyAsync(d_t, vt.data(), total * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
            r = deform_weights(d_npos, d_ntime, nn, d_in, kind, d_t, total, d_ids, d_w, s); if (r) return r;
            r = deform_apply(d_npos, d_x, nn, d_ids, d_w, d_in, d_out, kind, total, s); if (r) return r;
            off = 0;
            for (size_t i = 0; i < c->slices.size(); ++i) {
                const auto& sl = c->slices[i];
                const size_t cnt = kind == 0 ? (sl.has_processed ? sl.processed_count : 0) : (sl.has_mesh ? sl.mesh_nv : 0);
                if (!cnt) continue;
                void* h = c->deform_arena->alloc(cnt * rec);
                if (!h) { set_error("kt_deform_map: pinned host memory for %zu deformed records", cnt); return KT_ERR_CUDA; }
                KT_CUDA(cudaMemcpyAsync(h, (const char*)d_out + off * rec, cnt * rec, cudaMemcpyDeviceToHost, s));
                if (kind == 0) c->deformed[i].processed = (kt_point_xyzrgbnormal*)h; else c->deformed[i].mesh_verts = (kt_mesh_vertex*)h;
                off += cnt;
            }
            KT_CUDA(cudaStreamSynchronize(s));                                            // vt and the device buffers are reused
        }
        return 0;
    };
    const int r = run();
    cudaStreamSynchronize(c->stream);
    cleanup();
    if (r) c->deformed.clear();
    return r;
}


int kt_deform_map(kt_ctx* c, const kt_dense_pose* corrected, size_t n, const kt_deform_constraint* points, size_t n_points, float node_spacing,
                  kt_deform_report* report)
{
    if (!c || !report || (n && !corrected) || (n_points && !points) || !(node_spacing >= 0.f)) { set_error("kt_deform_map: bad argument"); return KT_ERR_INVALID; }
    std::memset(report, 0, sizeof(*report));
    if (c->world > 1) { set_error("kt_deform_map: a volume shared by %d GPUs cannot be deformed", c->world); return KT_ERR_INVALID; }
    std::vector<float> npos; std::vector<uint64_t> ntime;
    int r = deform_nodes(c, node_spacing, npos, ntime, "kt_deform_map"); if (r) return r;
    // constraints: corrected camera positions, then the caller's points
    const size_t nd = c->dense_poses.size();
    std::vector<float> gpos(nd * 3); std::vector<uint64_t> gtime(nd);
    for (size_t i = 0; i < nd; ++i) { gtime[i] = c->dense_poses[i].timestamp; for (int e = 0; e < 3; ++e) gpos[3 * i + e] = c->dense_poses[i].pose[4 * e + 3]; }
    std::vector<uint64_t> ctime(n); std::vector<double> cpos(3 * n);
    for (size_t i = 0; i < n; ++i) { ctime[i] = corrected[i].timestamp; for (int e = 0; e < 3; ++e) cpos[3 * i + e] = corrected[i].pose[4 * e + 3]; }
    std::vector<DeformConstraint> cons;
    const long miss = deform_pose_constraints(gtime.data(), gpos.data(), nd, ctime.data(), cpos.data(), n, cons);
    if (miss >= 0) { set_error("kt_deform_map: corrected pose %ld has timestamp %llu, which is not in the dense pose graph", miss, (unsigned long long)ctime[miss]); return KT_ERR_INVALID; }
    for (size_t i = 0; i < n_points; ++i) {
        DeformConstraint q; q.time = points[i].time;
        for (int e = 0; e < 3; ++e) { q.src[e] = points[i].source[e]; q.dst[e] = points[i].target[e]; }
        cons.push_back(q);
    }
    const size_t m = cons.size();
    if (!m) { set_error("kt_deform_map: no constraints"); return KT_ERR_INVALID; }
    for (size_t l = 0; l < m; ++l)
        if (deform_first_non_finite(cons[l].src, 3) >= 0 || deform_first_non_finite(cons[l].dst, 3) >= 0) {
            if (l < n) set_error("kt_deform_map: corrected pose %zu has a translation that is not finite", l);
            else set_error("kt_deform_map: point constraint %zu has a source or target that is not finite", l - n);
            return KT_ERR_INVALID;
        }
    return deform_run(c, npos, ntime, cons, report);
}

// Deformation::addCameraCamera + addCameraLoop (Deformation.cpp:130-346) with iSAMInterface (iSAMInterface.cpp:44-140): the pose graph of
// the dense poses, every accepted loop and the new one, optimised from the tracked trajectory on the GPU (kt_pgo.cu); the chi2 gate; on
// acceptance the map deformation of kt_deform_map.  Every check precedes any change of state.
int kt_close_loop(kt_ctx* c, const kt_loop_constraint* loop, float pose_spacing, float node_spacing, double isam_thresh, kt_loop_report* report)
{
    if (!c || !loop || !report || !(pose_spacing >= 0.f) || !(node_spacing >= 0.f) || !(isam_thresh > 0.0) ||
        (loop->n_inliers && (!loop->inliers1 || !loop->inliers2))) { set_error("kt_close_loop: bad argument"); return KT_ERR_INVALID; }
    std::memset(report, 0, sizeof(*report));
    if (c->world > 1) { set_error("kt_close_loop: a volume shared by %d GPUs cannot be loop-closed", c->world); return KT_ERR_INVALID; }
    if (c->loops.size() >= (size_t)PGO_MAX_LOOPS) { set_error("kt_close_loop: %zu loops accepted already, at most %d", c->loops.size(), PGO_MAX_LOOPS); return KT_ERR_CAPACITY; }
    if (loop->time1 == loop->time2) { set_error("kt_close_loop: time1 == time2"); return KT_ERR_INVALID; }
    const int chk = pgo_check_constraint(loop->constraint);
    if (chk) { set_error(chk == 1 ? "kt_close_loop: the constraint is not finite" : "kt_close_loop: the constraint's rotation is not orthonormal within 1e-3"); return KT_ERR_INVALID; }
    if (deform_first_non_finite(loop->inliers1, 3 * loop->n_inliers) >= 0 || deform_first_non_finite(loop->inliers2, 3 * loop->n_inliers) >= 0) {
        set_error("kt_close_loop: an inlier is not finite"); return KT_ERR_INVALID;
    }
    const size_t nd = c->dense_poses.size();
    std::unordered_map<uint64_t, int> at;                         // the last dense pose with a timestamp (iSAM's std::map cameraNode)
    for (size_t i = 0; i < nd; ++i) at[c->dense_poses[i].timestamp] = (int)i;
    if (!at.count(loop->time1) || !at.count(loop->time2)) { set_error("kt_close_loop: time %llu is not in the dense pose graph",
        (unsigned long long)(at.count(loop->time1) ? loop->time2 : loop->time1)); return KT_ERR_INVALID; }
    bool map = false;
    for (const auto& sl : c->slices) if (sl.has_processed || sl.has_mesh) map = true;
    std::vector<float> npos; std::vector<uint64_t> ntime;
    if (map) { const int r = deform_nodes(c, node_spacing, npos, ntime, "kt_close_loop"); if (r) return r; }

    // the loops: accepted ones, then the new one
    std::vector<kt_ctx::Loop> loops = c->loops;
    { kt_ctx::Loop l; l.time1 = loop->time1; l.time2 = loop->time2; std::memcpy(l.C, loop->constraint, sizeof(l.C));
      l.in1.assign(loop->inliers1, loop->inliers1 + 3 * loop->n_inliers); l.in2.assign(loop->inliers2, loop->inliers2 + 3 * loop->n_inliers);
      loops.push_back(l); }
    // nodes (addCameraCamera)
    std::vector<float> gpos(nd * 3); std::vector<unsigned char> flagged(nd, 0);
    for (size_t i = 0; i < nd; ++i) { flagged[i] = c->dense_poses[i].is_loop_pose ? 1 : 0; for (int e = 0; e < 3; ++e) gpos[3 * i + e] = c->dense_poses[i].pose[4 * e + 3]; }
    for (const auto& l : loops) { flagged[at[l.time1]] = 1; flagged[at[l.time2]] = 1; }
    const std::vector<int> take = pgo_select_nodes(gpos.data(), flagged.data(), nd, pose_spacing);
    const int n = (int)take.size();
    if (n < 2) { set_error("kt_close_loop: the dense pose graph has %d poses", n); return KT_ERR_STATE; }
    if (n > PGO_MAX_NODES) { set_error("kt_close_loop: %d pose-graph nodes, at most %d (raise pose_spacing)", n, PGO_MAX_NODES); return KT_ERR_CAPACITY; }
    for (int k = 1; k < n; ++k)
        if (c->dense_poses[take[k]].timestamp <= c->dense_poses[take[k - 1]].timestamp) { set_error("kt_close_loop: the dense pose graph's timestamps are not ascending"); return KT_ERR_STATE; }
    std::unordered_map<int, int> node_of;
    for (int k = 0; k < n; ++k) node_of[take[k]] = k;
    // factors (cameraNode's prior, addCameraCameraConstraint, addLoopConstraint) and the initial estimate in the isam frame
    std::vector<double> X0(16 * (size_t)n);
    for (int k = 0; k < n; ++k) pgo_pose_to_isam(c->dense_poses[take[k]].pose, &X0[16 * (size_t)k]);
    std::vector<PgoFactor> f(n + loops.size());
    f[0].i = -1; f[0].j = 0; pgo_vector(&X0[0], f[0].z);
    for (int k = 1; k < n; ++k) { f[k].i = k - 1; f[k].j = k; pgo_odometry_z(c->dense_poses[take[k - 1]].pose, c->dense_poses[take[k]].pose, f[k].z); }
    for (size_t l = 0; l < loops.size(); ++l) {
        PgoFactor& q = f[n + l];
        q.i = node_of[at[loops[l].time1]]; q.j = node_of[at[loops[l].time2]];
        pgo_loop_z(loops[l].C, q.z);
    }

    KT_CUDA(cudaSetDevice(c->cfg.device));
    double* d_X = 0;
    KT_CUDA(cudaMalloc((void**)&d_X, X0.size() * sizeof(double)));
    std::vector<double> X(X0.size());
    kt_pgo_report pr;
    int r = 0;
    if (!(r = kt::cuda_check(cudaMemcpyAsync(d_X, X0.data(), X0.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream), "upload", __FILE__, __LINE__)))
        r = pgo_optimise(d_X, n, f.data(), (int)f.size(), d_X, &pr, c->stream);
    if (!r) r = kt::cuda_check(cudaMemcpy(X.data(), d_X, X.size() * sizeof(double), cudaMemcpyDeviceToHost), "download", __FILE__, __LINE__);
    cudaFree(d_X);
    if (r) return r;
    report->nodes = pr.nodes; report->factors = pr.factors; report->loops = pr.loops; report->iterations = pr.iterations;
    report->chi2_initial = pr.chi2_initial; report->chi2_final = pr.chi2_final; report->solver_failed = pr.solver_failed;
    report->accepted = !pr.solver_failed && pr.chi2_final < isam_thresh;          // Deformation.cpp:256
    if (!report->accepted) return KT_OK;                                            // :336-343: nothing observable changes

    // the optimised nodes in the world frame
    std::vector<kt_dense_pose> nodes(n);
    std::vector<double> Pw(16 * (size_t)n);
    for (int k = 0; k < n; ++k) {
        pgo_pose_from_isam(&X[16 * (size_t)k], &Pw[16 * (size_t)k]);
        nodes[k].timestamp = c->dense_poses[take[k]].timestamp; nodes[k].is_loop_pose = flagged[take[k]];
        for (int q = 0; q < 16; ++q) nodes[k].pose[q] = (float)Pw[16 * (size_t)k + q];
    }
    if (map) {
        // one position constraint per node, one point constraint per inlier of every accepted loop (addCameraLoop :192-315)
        std::vector<DeformConstraint> cons;
        for (int k = 0; k < n; ++k) {
            DeformConstraint q; q.time = nodes[k].timestamp;
            for (int e = 0; e < 3; ++e) { q.src[e] = c->dense_poses[take[k]].pose[4 * e + 3]; q.dst[e] = Pw[16 * (size_t)k + 4 * e + 3]; }
            cons.push_back(q);
        }
        for (const auto& l : loops)
            for (int side = 0; side < 2; ++side) {
                const uint64_t t = side ? l.time2 : l.time1;
                const std::vector<float>& in = side ? l.in2 : l.in1;
                const float* Pt = c->dense_poses[at[t]].pose;
                const double* Po = &Pw[16 * (size_t)node_of[at[t]]];
                for (size_t p = 0; p + 2 < in.size(); p += 3) {
                    DeformConstraint q; q.time = t;
                    for (int e = 0; e < 3; ++e) {
                        q.src[e] = (float)((double)Pt[4 * e] * in[p] + (double)Pt[4 * e + 1] * in[p + 1] + (double)Pt[4 * e + 2] * in[p + 2] + (double)Pt[4 * e + 3]);
                        q.dst[e] = Po[4 * e] * in[p] + Po[4 * e + 1] * in[p + 1] + Po[4 * e + 2] * in[p + 2] + Po[4 * e + 3];
                    }
                    cons.push_back(q);
                }
            }
        // A CUDA error here drops the deformed copies, as kt_deform_map does, and the loop is not recorded: the loops and the corrected
        // trajectory stay those of the last accepted loop, and the next accepted loop deforms the original slices again.
        r = deform_run(c, npos, ntime, cons, &report->deform);
        if (r) return r;
        report->map_deformed = report->deform.deformed;
    }
    c->loops.swap(loops);
    c->pgo_nodes.swap(nodes);
    return KT_OK;
}

int kt_num_loops(kt_ctx* c) { return c ? (int)c->loops.size() : 0; }
int kt_num_pose_graph_nodes(kt_ctx* c) { return c ? (int)c->pgo_nodes.size() : 0; }
int kt_get_pose_graph_node(kt_ctx* c, int idx, kt_dense_pose* out)
{
    if (!c || !out || idx < 0 || idx >= (int)c->pgo_nodes.size()) { set_error("kt_get_pose_graph_node: bad index"); return KT_ERR_INVALID; }
    *out = c->pgo_nodes[idx];
    return KT_OK;
}

int kt_get_deformed_slice(kt_ctx* c, int idx, kt_point_xyzrgbnormal* points, size_t max_points, size_t* count)
{
    if (!c || idx < 0 || idx >= (int)c->slices.size()) { set_error("kt_get_deformed_slice: bad index"); return KT_ERR_INVALID; }
    if (idx >= (int)c->deformed.size()) { set_error("kt_get_deformed_slice: slice %d was recorded after the last kt_deform_map", idx); return KT_ERR_STATE; }
    const SliceRec& s = c->slices[idx];
    if (!s.has_processed) { set_error("kt_get_deformed_slice: slice %d was recorded with slice processing off (kt_set_slice_processing)", idx); return KT_ERR_STATE; }
    if (count) *count = s.processed_count;
    const size_t n = std::min(max_points, s.processed_count);
    if (points && n) std::memcpy(points, c->deformed[idx].processed, n * sizeof(kt_point_xyzrgbnormal));
    return KT_OK;
}

int kt_get_deformed_slice_mesh(kt_ctx* c, int idx, kt_mesh_vertex* verts, size_t max_verts, size_t* n_verts)
{
    if (!c || idx < 0 || idx >= (int)c->slices.size()) { set_error("kt_get_deformed_slice_mesh: bad index"); return KT_ERR_INVALID; }
    if (idx >= (int)c->deformed.size()) { set_error("kt_get_deformed_slice_mesh: slice %d was recorded after the last kt_deform_map", idx); return KT_ERR_STATE; }
    const SliceRec& s = c->slices[idx];
    if (!s.has_mesh) { set_error("kt_get_deformed_slice_mesh: slice %d was recorded with meshing off (kt_set_slice_meshing)", idx); return KT_ERR_STATE; }
    if (n_verts) *n_verts = s.mesh_nv;
    const size_t n = std::min(max_verts, s.mesh_nv);
    if (verts && n) std::memcpy(verts, c->deformed[idx].mesh_verts, n * sizeof(kt_mesh_vertex));
    return KT_OK;
}

int kt_save_deformed_mesh_ply(kt_ctx* c, const char* path)
{
    if (!c || !path) return KT_ERR_INVALID;
    if (c->deformed.empty()) { set_error("kt_save_deformed_mesh_ply: no kt_deform_map since the last reset"); return KT_ERR_STATE; }
    return save_mesh_ply(c, path, c->deformed.size(), true, "kt_save_deformed_mesh_ply");
}

int kt_get_slice_info(kt_ctx* c, int idx, kt_slice_info* info)
{
    if (!c || !info || idx < 0 || idx >= (int)c->slices.size()) { set_error("kt_get_slice_info: bad argument"); return KT_ERR_INVALID; }
    const SliceRec& s = c->slices[idx];
    info->dimension = s.dimension;
    info->odometry = c->cfg.odometry == 0 ? 0 : 2;            // CloudSlice::ICP / CloudSlice::RGBD
    for (int i = 0; i < 3; ++i) info->camera_t[i] = s.camera_t[i];
    for (int i = 0; i < 9; ++i) info->camera_R[i] = s.camera_R[i];
    info->utime = s.utime;
    info->count = s.count;
    return KT_OK;
}

int kt_get_trace(kt_ctx* c, float* dst, int max_iters, int* n_iters)
{
    if (!c) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    int n = std::min(max_iters, c->trace_iters);
    if (n_iters) *n_iters = c->trace_iters;
    if (dst && n > 0) {
        KT_CUDA(cudaMemcpyAsync(c->trace_host, c->trace_dev, (size_t)n * TRACE_STRIDE * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        KT_CUDA(cudaStreamSynchronize(c->stream));
        std::memcpy(dst, c->trace_host, (size_t)n * TRACE_STRIDE * sizeof(float));
    }
    return KT_OK;
}

int kt_volume_export_reference_layout(kt_ctx* c, int16_t* tsdf_host, uint8_t* color_host)
{
    if (!c) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    KT_CUDA(cudaStreamSynchronize(c->stream));
    const size_t plane = (size_t)c->cfg.vol * c->cfg.vol;
    if (c->world == 1) {
        if (tsdf_host) KT_CUDA(cudaMemcpy(tsdf_host, c->tsdf, plane * c->cfg.vol * 2, cudaMemcpyDeviceToHost));
        if (color_host) KT_CUDA(cudaMemcpy(color_host, c->color, plane * c->cfg.vol * 4, cudaMemcpyDeviceToHost));
        return KT_OK;
    }
    // shared volume: the storage planes this rank OWNS, in local plane order (kt_mgpu_info gives the block size; local plane l is storage
    // plane ((l / B * world + rank) * B + l % B); the TSDF planes are gathered out of the local replica
    if (color_host) KT_CUDA(cudaMemcpy(color_host, c->color, plane * c->local_planes * 4, cudaMemcpyDeviceToHost));
    if (tsdf_host) {
        const int B = c->mg_block;
        for (int l0 = 0; l0 < c->local_planes; l0 += B) {
            const size_t sz0 = (size_t)((l0 / B) * c->world + c->rank) * B;
            KT_CUDA(cudaMemcpy(tsdf_host + (size_t)l0 * plane, c->tsdf + sz0 * plane, plane * B * 2, cudaMemcpyDeviceToHost));
        }
    }
    return KT_OK;
}

int kt_download_map(kt_ctx* c, int which, int level, void* dst)
{
    if (!c || !dst || level < 0 || level >= LEVELS || which < 0 || which > 8) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const size_t Pl = ((size_t)c->cfg.rows * c->cfg.cols) >> (2 * level);
    const void* src = which == 0 ? (void*)c->vmaps_curr[level] : which == 1 ? (void*)c->nmaps_curr[level] :
                      which == 2 ? (void*)c->vmaps_g_prev[level] : which == 3 ? (void*)c->nmaps_g_prev[level] :
                      which == 4 ? (void*)c->depths_curr[level] : which == 5 ? (void*)c->vmap_curr_color :
                      which == 6 ? (void*)c->depth_scaled : which == 7 ? (void*)c->cw_scratch : (void*)c->rgbf_scratch;      // 6-8: integration inputs, level 0
    const size_t bytes = which <= 3 ? Pl * 12 : which == 4 ? Pl * 2 : which == 8 ? Pl * 16 : Pl * 4;
    KT_CUDA(cudaStreamSynchronize(c->stream));
    KT_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    return KT_OK;
}

int kt_set_stage_timing(kt_ctx* c, int enabled) { if (!c) return KT_ERR_INVALID; c->timing = enabled != 0; return KT_OK; }

int kt_get_stage_ms(kt_ctx* c, float* ms6)
{
    if (!c || !ms6) return KT_ERR_INVALID;
    if (!c->timing) { for (int i = 0; i < 6; ++i) ms6[i] = 0.f; return KT_OK; }
    KT_CUDA(cudaStreamSynchronize(c->stream));
    float total = 0.f;
    for (int i = 0; i < 5; ++i) { float t = 0.f; if (cudaEventElapsedTime(&t, c->ev[i], c->ev[i + 1]) != cudaSuccess) { cudaGetLastError(); t = 0.f; } ms6[i] = t; total += t; }
    ms6[5] = total;
    return KT_OK;
}

int kt_debug_icp_profile(kt_ctx* c, long long* out512)
{
    if (!c || !out512) return KT_ERR_INVALID;
    KT_CUDA(cudaStreamSynchronize(c->stream));
    KT_CUDA(cudaMemcpy(out512, c->prof_dev, 64 * 8 * sizeof(long long), cudaMemcpyDeviceToHost));
    return KT_OK;
}

int kt_mgpu_arena_handle(kt_ctx* c, void* handle64)
{
    if (!c || !handle64) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    cudaIpcMemHandle_t h;
    KT_CUDA(cudaIpcGetMemHandle(&h, c->arena));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    std::memcpy(handle64, &h, 64);
    return KT_OK;
}

int kt_mgpu_connect(kt_ctx* c, const void* handles, int n)
{
    if (!c || !handles || n != c->world) { set_error("kt_mgpu_connect: need exactly world handles"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    unsigned int* flags_host[MAX_GPUS];
    for (int g = 0; g < c->world; ++g) {
        if (g == c->rank) c->peer_arena[g] = c->arena;
        else {
            cudaIpcMemHandle_t h; std::memcpy(&h, (const char*)handles + (size_t)g * 64, 64);
            void* p = 0;
            KT_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
            c->peer_arena[g] = (uint8_t*)p;
        }
        c->vv.tsdf[g] = (int16_t*)(c->peer_arena[g] + c->off_tsdf);
        c->vv.color[g] = c->peer_arena[g] + c->off_color;
        flags_host[g] = (unsigned int*)(c->peer_arena[g] + c->off_flags);
    }
    for (int g = c->world; g < MAX_GPUS; ++g) flags_host[g] = flags_host[0];
    KT_CUDA(cudaMemcpy(c->peer_flags_dev, flags_host, sizeof(flags_host), cudaMemcpyHostToDevice));
    c->connected = true;
    return KT_OK;
}

int kt_mgpu_info(kt_ctx* c, int* info5)       // world, rank, colour planes owned, planes per ownership block, arena bytes (MB)
{
    if (!c || !info5) return KT_ERR_INVALID;
    info5[0] = c->world; info5[1] = c->rank; info5[2] = c->local_planes; info5[3] = c->mg_block; info5[4] = (int)(c->arena_bytes >> 20);
    return KT_OK;
}

int kt_mgpu_export_tsdf_replica(kt_ctx* c, int16_t* tsdf_host)      // the full local TSDF replica, storage order (test tap)
{
    if (!c || !tsdf_host) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    KT_CUDA(cudaStreamSynchronize(c->stream));
    KT_CUDA(cudaMemcpy(tsdf_host, c->tsdf, (size_t)c->cfg.vol * c->cfg.vol * c->cfg.vol * 2, cudaMemcpyDeviceToHost));
    return KT_OK;
}

float kt_get_icp_kernel_ms(kt_ctx* c)
{
    if (!c || !c->timing) return 0.f;
    cudaStreamSynchronize(c->stream);
    float t = 0.f;
    if (cudaEventElapsedTime(&t, c->ev_icp[0], c->ev_icp[1]) != cudaSuccess) { cudaGetLastError(); return 0.f; }
    return t;
}

int kt_get_kernel_ms(kt_ctx* c, float* ms3)
{
    if (!c || !ms3) return KT_ERR_INVALID;
    ms3[0] = ms3[1] = ms3[2] = 0.f;
    if (!c->timing) return KT_OK;
    cudaStreamSynchronize(c->stream);
    if (cudaEventElapsedTime(&ms3[0], c->ev_icp[0], c->ev_icp[1]) != cudaSuccess) { cudaGetLastError(); ms3[0] = 0.f; }
    if (cudaEventElapsedTime(&ms3[1], c->ev_krn[0], c->ev_krn[1]) != cudaSuccess) { cudaGetLastError(); ms3[1] = 0.f; }
    if (cudaEventElapsedTime(&ms3[2], c->ev_krn[2], c->ev_krn[3]) != cudaSuccess) { cudaGetLastError(); ms3[2] = 0.f; }
    return KT_OK;
}

int kt_span_mark(kt_ctx* c, int which)
{
    if (!c || which < 0 || which > 1) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    KT_CUDA(cudaEventRecord(c->ev_span[which], c->stream));
    return KT_OK;
}

float kt_span_elapsed_ms(kt_ctx* c)
{
    if (!c || cudaSetDevice(c->cfg.device) != cudaSuccess) return -1.f;
    float t = 0.f;
    if (cudaEventSynchronize(c->ev_span[1]) != cudaSuccess || cudaEventElapsedTime(&t, c->ev_span[0], c->ev_span[1]) != cudaSuccess) { cudaGetLastError(); return -1.f; }
    return t;
}

// ---- OdometryProvider at the ABI (OdometryProvider.h:42-52): one call = ICPOdometry / RGBDOdometry::getIncrementalTransformation
// (ICPOdometry.cpp:68-186, RGBDOdometry.cpp:165-393) on the whole-frame kernels, for a caller that owns the pose history and the maps (the
// reference's KintinuousTracker, or a fork of it).  The context only lends its odometry scratch and, for the photometric modes, keeps the
// last / next pyramids between calls like the RGBDOdometry object does.
int kt_odometry_first_run(kt_ctx* c, const uint16_t* depth_dev, const uint8_t* rgb_dev)             // RGBDOdometry::firstRun (RGBDOdometry.cpp:160-163)
{
    if (!c || !depth_dev || !rgb_dev) { set_error("kt_odometry_first_run: null argument"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    if (c->cfg.odometry == 0) return KT_OK;
    FrontendArgs fa; std::memset(&fa, 0, sizeof(fa));
    fa.depth_raw = depth_dev; fa.rgb = rgb_dev; fa.rows = c->cfg.rows; fa.cols = c->cfg.cols; fa.k.fx = c->cfg.fx; fa.k.fy = c->cfg.fy; fa.k.cx = c->cfg.cx; fa.k.cy = c->cfg.cy;
    fa.depths = c->depths_curr; fa.cut_off = 6000; fa.depth_m = c->lastDepth; fa.intensity = c->lastImage; fa.dIdx = c->nextdIdx; fa.dIdy = c->nextdIdy;
    int r = frontend_pyramid(fa, c->stream); if (r) return r;
    KT_CUDA(cudaStreamSynchronize(c->stream));
    return KT_OK;
}

int kt_odometry_increment(kt_ctx* c, const uint16_t* depth_dev, const uint8_t* rgb_dev, const float* Rprev9, const float* tprev3,
                          const float* const* vmaps_g_prev4, const float* const* nmaps_g_prev4,
                          const float* const* vmaps_curr4, const float* const* nmaps_curr4, float* Rcurr9, float* tcurr3)
{
    if (!c || !Rprev9 || !tprev3 || !vmaps_g_prev4 || !nmaps_g_prev4 || !Rcurr9 || !tcurr3) { set_error("kt_odometry_increment: null argument"); return KT_ERR_INVALID; }
    if ((!vmaps_curr4 || !nmaps_curr4 || c->cfg.odometry != 0) && (!depth_dev || !rgb_dev)) { set_error("kt_odometry_increment: this mode needs the depth / colour frame"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    int r;
    float* keep[4][LEVELS];
    for (int l = 0; l < LEVELS; ++l) { keep[0][l] = c->vmaps_g_prev[l]; keep[1][l] = c->nmaps_g_prev[l]; keep[2][l] = c->vmaps_curr[l]; keep[3][l] = c->nmaps_curr[l]; }
    auto restore = [&]() { for (int l = 0; l < LEVELS; ++l) { c->vmaps_g_prev[l] = keep[0][l]; c->nmaps_g_prev[l] = keep[1][l]; c->vmaps_curr[l] = keep[2][l]; c->nmaps_curr[l] = keep[3][l]; } };
    if (vmaps_curr4 && nmaps_curr4) {
        // the caller's current maps (createVMap / createNMap of its own pyramid); the photometric set still comes from the frame
        if (c->cfg.odometry != 0) {
            FrontendArgs fa; std::memset(&fa, 0, sizeof(fa));
            fa.depth_raw = depth_dev; fa.rgb = rgb_dev; fa.rows = c->cfg.rows; fa.cols = c->cfg.cols; fa.k.fx = c->cfg.fx; fa.k.fy = c->cfg.fy; fa.k.cx = c->cfg.cx; fa.k.cy = c->cfg.cy;
            fa.depths = c->depths_curr; fa.cut_off = 6000; fa.depth_m = c->nextDepth; fa.intensity = c->nextImage; fa.dIdx = c->nextdIdx; fa.dIdy = c->nextdIdy;
            if ((r = frontend_pyramid(fa, c->stream))) return r;
        }
        for (int l = 0; l < LEVELS; ++l) { c->vmaps_curr[l] = const_cast<float*>(vmaps_curr4[l]); c->nmaps_curr[l] = const_cast<float*>(nmaps_curr4[l]); }
    } else {
        if ((r = build_frontend(c, depth_dev, rgb_dev, c->depth_scaled, c->depths_curr, c->vmaps_curr, c->nmaps_curr, 0, 0, c->cw_scratch, c->rgbf_scratch,
                                c->cfg.odometry != 0 ? c->nextDepth : 0, c->cfg.odometry != 0 ? c->nextImage : 0, c->stream))) return r;
    }
    for (int l = 0; l < LEVELS; ++l) { c->vmaps_g_prev[l] = const_cast<float*>(vmaps_g_prev4[l]); c->nmaps_g_prev[l] = const_cast<float*>(nmaps_g_prev4[l]); }
    M3 Rp, Rc; V3 tp, tc;
    for (int k = 0; k < 9; ++k) Rp.m[k] = Rprev9[k];
    for (int k = 0; k < 3; ++k) tp.v[k] = tprev3[k];
    Rc = Rp; tc = tp;
    const bool fr = c->frontend_ready; c->frontend_ready = true;          // the front end of this call is already built
    r = run_odometry(c, Rp, tp, &Rc, &tc);
    c->frontend_ready = fr;
    restore();
    if (r) return r;
    for (int k = 0; k < 9; ++k) Rcurr9[k] = Rc.m[k];
    for (int k = 0; k < 3; ++k) tcurr3[k] = tc.v[k];
    return KT_OK;
}

// getLiveImage (KintinuousTracker.cpp:835-862, 960-981, 1125-1154): shaded weight image, colour image and model depth of the predicted
// surface at the last pose.  One launch on the tracker's stream + one copy; any output may be NULL.
int kt_get_live_image(kt_ctx* c, uint8_t* shaded_rgb_host, uint8_t* color_rgb_host, uint16_t* model_depth_host)
{
    if (!c) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    if (!c->view_dev) { int r = dev_alloc(c, &c->view_dev, P * 8); if (r) return r; }
    uint8_t* shaded = c->view_dev; uint8_t* col = c->view_dev + P * 3; uint16_t* dep = (uint16_t*)(c->view_dev + P * 6);
    const float light[3] = {c->size * -3.f, c->size * -3.f, c->size * -3.f};
    const M3 Rinv = m3_inverse(c->rmats.back());
    int r = generate_views(c->vmaps_g_prev[0], c->nmaps_g_prev[0], c->vmap_curr_color, c->cfg.rows, c->cfg.cols, light, 1,
                           shaded_rgb_host ? shaded : 0, color_rgb_host ? col : 0, Rinv.m, c->tvecs.back().v, model_depth_host ? dep : 0, c->stream);
    if (r) return r;
    if (shaded_rgb_host) KT_CUDA(cudaMemcpyAsync(shaded_rgb_host, shaded, P * 3, cudaMemcpyDeviceToHost, c->stream));
    if (color_rgb_host) KT_CUDA(cudaMemcpyAsync(color_rgb_host, col, P * 3, cudaMemcpyDeviceToHost, c->stream));
    if (model_depth_host) KT_CUDA(cudaMemcpyAsync(model_depth_host, dep, P * 2, cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(cudaStreamSynchronize(c->stream));
    return KT_OK;
}

// getLiveTsdf (KintinuousTracker.cpp:835-850, 1087-1123): the whole volume's surface points without recording a slice.
int kt_get_live_tsdf(kt_ctx* c, kt_point_xyzrgb* points, size_t max_points, size_t* count)
{
    if (!c) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    int vWrapCopy[3]; vwrap_copy(c, vWrapCopy);
    const int V = c->cfg.vol;
    int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
    int r = fetch_cloud(c, vWrapCopy, lo, hi);
    if (r) return r;
    if (count) *count = c->cloud_count;
    const size_t n = std::min(max_points, c->cloud_count);
    if (points && n) KT_CUDA(cudaMemcpy(points, c->cloud_dev, n * sizeof(kt_point_xyzrgb), cudaMemcpyDeviceToHost));
    return KT_OK;
}

int kt_debug_last_integrate(kt_ctx* c, float* Rinv9, float* t3, int* wrap3)
{
    if (!c || !Rinv9 || !t3 || !wrap3) return KT_ERR_INVALID;
    for (int k = 0; k < 9; ++k) Rinv9[k] = c->last_int_Rinv[k];
    for (int k = 0; k < 3; ++k) { t3[k] = c->last_int_t[k]; wrap3[k] = c->last_int_wrap[k]; }
    return KT_OK;
}

long long kt_launch_count(kt_ctx* c) { return c ? g_launches.load() - c->launches_at_create : g_launches.load(); }

int kt_alloc_pinned(void** ptr, size_t bytes) { KT_CUDA(cudaMallocHost(ptr, bytes)); return KT_OK; }
int kt_free_pinned(void* ptr) { if (ptr) KT_CUDA(cudaFreeHost(ptr)); return KT_OK; }

} // extern "C"
