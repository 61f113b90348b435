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
#include "kt_place.hpp"
#include <cstdlib>
#include "../../include/kintinuous_b200.h"
#include <memory>
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
                  unsigned long long* mesh_vkeys; unsigned long long* mesh_tcells; MeshKeyFrame mesh_frame;    // local keys: kt_get_slice_mesh_keys
                  Event ready; float camera_t[3]; float camera_R[9]; uint64_t utime; };

// Pinned host memory handed out in slabs (one allocation per 64 MB, not per slice); kt_reset rewinds it, the slabs live as long as it.
struct PinnedArena {
    Allocations slabs; std::vector<std::pair<char*, size_t> > chunks; size_t chunk_used; size_t current;
    PinnedArena() : chunk_used(0), current(0) {}
    void* alloc(size_t bytes)
    {
        bytes = (bytes + 255) & ~(size_t)255;
        while (current < chunks.size() && chunk_used + bytes > chunks[current].second) { ++current; chunk_used = 0; }
        if (current >= chunks.size()) {
            const size_t sz = std::max(bytes, (size_t)64 << 20);
            char* q = 0;
            if (slabs.pinned(&q, sz, "a pinned arena slab")) return 0;
            chunks.push_back(std::make_pair(q, sz));
            current = chunks.size() - 1; chunk_used = 0;
        }
        void* r = chunks[current].first + chunk_used;
        chunk_used += bytes;
        return r;
    }
    void rewind() { current = 0; chunk_used = 0; }
};

// The buffer sets of one frame, each swapped whole.  alloc() gives every buffer of the set for an image of P pixels, owned by `mem`.
struct MapPyramid {            // the filtered depth pyramid and the vertex / normal maps (planar x, y, z) of every level
    uint16_t* depths[LEVELS]; float* vmaps[LEVELS]; float* nmaps[LEVELS];
    int alloc(Allocations& mem, size_t P, const char* what)
    {
        for (size_t l = 0, Pl = P; l < LEVELS; ++l, Pl /= 4)
            if (mem.device(&depths[l], Pl, what) || mem.device(&vmaps[l], Pl * 3, what) || mem.device(&nmaps[l], Pl * 3, what)) return KT_ERR_CUDA;
        return 0;
    }
};
struct FrameInputs {           // the raw frame as copied in
    uint16_t* depth; uint8_t* rgb;
    int alloc(Allocations& mem, size_t P, const char* what) { return mem.device(&depth, P, what) || mem.device(&rgb, P * 3, what) ? KT_ERR_CUDA : 0; }
};
struct FrontEnd {              // everything build_frontend writes that does not depend on the pose
    float* depth_scaled; MapPyramid maps; float* cw; float* rgbf;
    int alloc(Allocations& mem, size_t P, const char* what)
    {
        return mem.device(&depth_scaled, P, what) || maps.alloc(mem, P, what) || mem.device(&cw, P, what) || mem.device(&rgbf, P * 4, what) ? KT_ERR_CUDA : 0;
    }
};
struct PhotometricPyramid {    // one of the photometric odometry's last / next sets (RGBDOdometry's lastDepth / lastImage, nextDepth / nextImage)
    float* depth[LEVELS]; uint8_t* image[LEVELS];
    int alloc(Allocations& mem, size_t P, const char* what)
    {
        for (size_t l = 0, Pl = P; l < LEVELS; ++l, Pl /= 4) if (mem.device(&depth[l], Pl, what) || mem.device(&image[l], Pl, what)) return KT_ERR_CUDA;
        return 0;
    }
};

// what the host reads back after the odometry of a frame
struct OdomResult { float Rcurr[9]; float tcurr[3]; int timeout; unsigned int seq; int pad[2]; };     // seq: written last by the odometry kernel (mapped host memory)

// Place recognition (kt_set_loop_detection / kt_detect_loops): keyframes' raw depth, SURF keypoints / descriptors and their 3-D points, captured on
// `stream` (the frame path never waits for it on the host), and the scratch of the detection chain.  Allocated only while detection is on.
struct PlaceStore {
    Allocations mem;
    kt_loop_detection_params p;
    int rows, cols, maxK, maxF;
    cudaStream_t stream; cudaEvent_t ev_input, ev_copied;
    uint16_t* depth; uint8_t* rgb; float* kp; float* desc; float* xyz; int* nfeat_dev; int* nfeat_host;
    SurfWorkspace surf_ws;
    std::vector<uint64_t> times; std::vector<int> dense_idx;
    size_t processed; bool full;
    float lastR[9], lastG[3];
    uint64_t last_loop;
    // detection scratch
    int* best; float* d1; float* d2; unsigned char* pass; int* seg_passes;
    float* pn; float* po; float* uv; double* pose; unsigned char* inl; int* ninl; PnpWorkspace pnp_ws;
    MapPyramid maps[2];
    OdomState* state; unsigned long long* xwords; float* trace;
    kt_point_xyzrgb* cloud[2]; kt_point_xyzrgbnormal* cent[2]; double* d2fit; SliceWorkspace ws[2];
    std::vector<std::vector<float> > in_new, in_old;      // inliers of the results of the last kt_detect_loops
    ~PlaceStore() { if (stream) cudaStreamSynchronize(stream); }
};

} // namespace kt

using namespace kt;

struct kt_ctx {
    kt_config cfg;
    cudaStream_t stream;
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
    // this frame's inputs and front end; kt_prefetch_frame copies the NEXT frame into the spare sets and builds its front end there on a
    // side stream, overlapping the integrate / ray-cast of the frame before (they leave issue slots idle)
    FrameInputs in, in_spare; FrontEnd fe, fe_spare;
    const void* pf_depth; const void* pf_rgb; bool pf_valid;
    bool pf_built;             // the prefetched set holds the finished front end
    bool frontend_ready;       // set for the duration of one process_frame_device call
    cudaStream_t stream_copy; cudaEvent_t ev_prefetch, ev_done[2], ev_maps; int last_parity; bool maps_on_stream;   // ev_maps: this frame's front end (on `stream`) has written the current maps
    float* vmaps_g_prev[LEVELS]; float* nmaps_g_prev[LEVELS];
    uint8_t* vmap_curr_color; float* ztable;
    unsigned long long* xwords_dev; bool xwords_clean;      // exchange words of the whole-frame odometry kernels; zero between frames
    OdomState* state; float* partials; int* ipartials; float* trace_dev; float* pose12_dev; long long* prof_dev;
    kt_point_xyzrgb* cloud_dev; unsigned int* counter_dev; size_t cloud_capacity; size_t cloud_count;
    // slice hand-off: pinned arena, asynchronous download on stream_slices; ev_cloud_free = the last download has left cloud_dev / proc_dev
    PinnedArena slice_arena; cudaStream_t stream_slices; cudaEvent_t ev_cloud_ready, ev_cloud_free; bool cloud_busy;
    // CloudSliceProcessor on the device (kt_slice.cu): weight cull + voxel grid + normals of every slice before it leaves the GPU
    int slice_processing, slice_weight_cull; SliceWorkspace slice_ws; DeviceBuffer<kt_point_xyzrgbnormal> proc; size_t proc_count;
    // marching cubes of every slice's box before it is cleared (kt_mesh.cu); buffers grow at a shift, downloaded with the slice
    int slice_meshing, mesh_weight_cull; MeshWorkspace mesh_ws; DeviceBuffer<kt_mesh_vertex> mesh_verts; DeviceBuffer<uint32_t> mesh_tris;
    size_t mesh_nv, mesh_nt;
    DeviceBuffer<unsigned long long> mesh_vkeys, mesh_tcells; MeshKeyFrame mesh_frame;     // the slice mesh's local keys (mesh_emit) and their frame
    // the map as deformed by the last kt_deform_map (kt_deform.cu): one record per slice recorded before that call, in its own pinned
    // arena, or the slice's own buffers when the call left the map unchanged
    struct Deformed { kt_point_xyzrgbnormal* processed; kt_mesh_vertex* mesh_verts; };
    std::vector<Deformed> deformed; PinnedArena deform_arena;
    // loop closure (kt_close_loop, kt_pgo.cu): the accepted loops with their inliers, and the optimised nodes of the last accepted one
    struct Loop { uint64_t time1, time2; double C[16]; std::vector<float> in1, in2; };
    std::vector<Loop> loops; std::vector<kt_dense_pose> pgo_nodes;
    // the last correction of that deformation (kt_get_map_cloud's corrected map moves later slices by P_corr P_tracked^-1): the pose at
    // `time` as tracked and as corrected (the last corrected pose of kt_deform_map, the last pose-graph node of kt_close_loop)
    struct MapCorrection { uint64_t time; float tracked[16]; float corrected[16]; };
    MapCorrection map_corr;
    // RGB-D
    PhotometricPyramid ph_last, ph_next;
    int16_t* nextdIdx[LEVELS]; int16_t* nextdIdy[LEVELS]; float* pointClouds[LEVELS]; void* corresImg[LEVELS];
    // pinned host staging
    float* pose12_host; OdomResult* result_host; float* result_dev_alias; unsigned int pose_seq; float* trace_host; unsigned int* counter_host;
    int trace_iters; int shifted_last;
    // timing
    bool timing; cudaEvent_t ev[6]; cudaEvent_t ev_icp[2]; cudaEvent_t ev_krn[4]; cudaEvent_t ev_span[2];     // ev_krn: integrate / raycast launches alone (without the cross-GPU barriers the stage timers include)
    long long launches_at_create;
    Allocations mem;           // device and pinned buffers, events and streams created with the context
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
    DeviceBuffer<uint8_t> view;                                         // GUI taps: shaded image, colour image, model depth (allocated on first use)
    std::unique_ptr<PlaceStore> place;                                  // loop detection (null while it is off)
    std::unique_ptr<MapVolume> mapvol;                                  // the map volume (kt_mapvol.cu; null while it is off)
    bool mapvol_restore = false;                                        // the map volume refills the planes a shift clears
    // what member destructors cannot do: wait for the streams, unmap the peers' arenas, close the pose log
    ~kt_ctx()
    {
        cudaSetDevice(cfg.device);
        for (cudaStream_t s : {stream, stream_copy, stream_slices}) if (s) cudaStreamSynchronize(s);
        for (int g = 0; g < MAX_GPUS; ++g) if (peer_arena[g] && peer_arena[g] != arena) cudaIpcCloseMemHandle(peer_arena[g]);
        if (pose_log) fclose(pose_log);
    }
};

namespace {

const int MAX_TRACE_ITERS = 64;

void vwrap_copy(const kt_ctx* c, int* w)       // KintinuousTracker::vWrapCopyUpdate (.cpp:1075-1085)
{
    vwrap_nonneg(c->voxelWrap, c->cfg.vol, w);
}

// The last slice's asynchronous download (push_slice) may still be reading cloud_dev, proc and the mesh buffers: their writers wait.
int wait_slice_download(kt_ctx* c)
{
    if (c->cloud_busy) { KT_CUDA(cudaStreamWaitEvent(c->stream, c->ev_cloud_free, 0)); c->cloud_busy = false; }
    return 0;
}

int fetch_cloud(kt_ctx* c, const int* lo, const int* hi)      // TsdfVolume::fetchCloud (TSDFVolume.cpp:131-172)
{
    int vWrapCopy[3]; vwrap_copy(c, vWrapCopy);
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

// Marching cubes over the box [lo, hi) of the volume as it stands, on the tracker stream, into the context's mesh buffers (grown here:
// the count is read back first, once).  MeshGenerator::calculateMesh (MeshGenerator.cpp:193-227) on the device, by a different
// algorithm (kt_mesh.cu).
// keyed: a slice mesh, whose local vertex keys and triangle cells go to the context's key buffers as well (no extra launch).
int mesh_box(kt_ctx* c, const int* lo, const int* hi, bool keyed)
{
    MeshArgs a;
    int vWrapCopy[3]; vwrap_copy(c, vWrapCopy);
    a.tsdf = c->tsdf; a.color = c->color; a.vol = c->cfg.vol; a.volume_size = make_float3(c->size, c->size, c->size);
    a.wrap = make_int3(vWrapCopy[0], vWrapCopy[1], vWrapCopy[2]); a.real_wrap = make_int3(c->voxelWrap[0], c->voxelWrap[1], c->voxelWrap[2]);
    a.minX = lo[0]; a.maxX = hi[0]; a.minY = lo[1]; a.maxY = hi[1]; a.minZ = lo[2]; a.maxZ = hi[2]; a.weight_cull = c->mesh_weight_cull;
    size_t nv = 0, nt = 0;
    int r = mesh_count(a, &c->mesh_ws, &nv, &nt, c->stream); if (r) return r;
    if (nv > c->mesh_verts.capacity() || 3 * nt > c->mesh_tris.capacity() || (keyed && (nv > c->mesh_vkeys.capacity() || nt > c->mesh_tcells.capacity()))) {
        KT_CUDA(cudaStreamSynchronize(c->stream_slices));
        if ((r = c->mesh_verts.grow(nv, nv + nv / 4 + 1024, "slice mesh vertices")) ||
            (r = c->mesh_tris.grow(3 * nt, 3 * (nt + nt / 4 + 1024), "slice mesh triangles"))) return r;
        if (keyed && ((r = c->mesh_vkeys.grow(nv, nv + nv / 4 + 1024, "slice mesh vertex keys")) ||
                      (r = c->mesh_tcells.grow(nt, nt + nt / 4 + 1024, "slice mesh triangle cells")))) return r;
    }
    r = mesh_emit(a, &c->mesh_ws, nv, c->mesh_verts.get(), c->mesh_tris.get(), c->stream, keyed ? c->mesh_vkeys.get() : nullptr,
                  keyed ? c->mesh_tcells.get() : nullptr);
    if (r) return r;
    c->mesh_nv = nv; c->mesh_nt = nt;
    if (keyed) c->mesh_frame = mesh_key_frame(a);
    return 0;
}

// Cut the box [lo, hi) out of the volume for a slice, before it is cleared: its surface points into cloud_dev and, with slice meshing
// on, its keyed mesh into the mesh buffers.  push_slice records them.
int cut_box(kt_ctx* c, const int* lo, const int* hi)
{
    int r;
    if ((r = wait_slice_download(c)) || (r = fetch_cloud(c, lo, hi))) return r;
    return c->slice_meshing ? mesh_box(c, lo, hi, true) : 0;
}

// mutexOutCloudBuffer (KintinuousTracker.cpp:1156-1208): record the extracted cloud as a CloudSlice.  The points go to pinned host
// memory with an ASYNCHRONOUS copy on a side stream -- the frame's clear / integrate / ray cast do not wait for it; readers of the slice
// do (kt_get_slice waits on the slice's event).  With slice processing on, the slice is culled, voxel-gridded and given normals on the
// device first (kt_slice.cu) and both clouds are handed out.
int push_slice(kt_ctx* c, int dimension)
{
    SliceRec s; s.dimension = dimension; s.points = 0; s.count = c->cloud_count; s.processed = 0; s.processed_count = 0; s.has_processed = false;
    s.has_mesh = c->slice_meshing != 0; s.mesh_verts = 0; s.mesh_tris = 0; s.mesh_vkeys = 0; s.mesh_tcells = 0; s.mesh_frame = c->mesh_frame;
    s.mesh_nv = s.has_mesh ? c->mesh_nv : 0; s.mesh_nt = s.has_mesh ? c->mesh_nt : 0;
    c->proc_count = 0;
    if (c->slice_processing && c->cloud_count) {
        int r = c->proc.grow(c->cloud_capacity, c->cloud_capacity, "processed slice");
        if (!r) r = process_slice(c->cloud_dev, c->cloud_count, c->slice_weight_cull, c->voxel, 20, c->proc.get(), c->cloud_capacity, &c->proc_count, &c->slice_ws, c->stream);
        if (r) return r;
    }
    s.has_processed = c->slice_processing != 0;
    s.processed_count = c->proc_count;
    struct Download { const void* src; size_t bytes; void** host; };       // host: the slice's pointer to the pinned copy of src
    const Download downloads[] = {{c->cloud_dev, c->cloud_count * sizeof(kt_point_xyzrgb), (void**)&s.points},
                                  {c->proc.get(), c->proc_count * sizeof(kt_point_xyzrgbnormal), (void**)&s.processed},
                                  {c->mesh_verts.get(), s.mesh_nv * sizeof(kt_mesh_vertex), (void**)&s.mesh_verts},
                                  {c->mesh_tris.get(), s.mesh_nt * 3 * sizeof(uint32_t), (void**)&s.mesh_tris},
                                  {c->mesh_vkeys.get(), s.mesh_nv * sizeof(unsigned long long), (void**)&s.mesh_vkeys},
                                  {c->mesh_tcells.get(), s.mesh_nt * sizeof(unsigned long long), (void**)&s.mesh_tcells}};
    if (c->cloud_count || s.mesh_nv) {
        for (const Download& d : downloads)
            if (d.bytes && !(*d.host = c->slice_arena.alloc(d.bytes))) { set_error("pinned host memory for a slice of %zu points", c->cloud_count); return KT_ERR_CUDA; }
        int r = make_event(&s.ready, cudaEventDisableTiming, "slice download"); if (r) return r;
        KT_CUDA(cudaEventRecord(c->ev_cloud_ready, c->stream));
        KT_CUDA(cudaStreamWaitEvent(c->stream_slices, c->ev_cloud_ready, 0));
        for (const Download& d : downloads) if (d.bytes) KT_CUDA(cudaMemcpyAsync(*d.host, d.src, d.bytes, cudaMemcpyDeviceToHost, c->stream_slices));
        KT_CUDA(cudaEventRecord(s.ready.get(), c->stream_slices));
        KT_CUDA(cudaEventRecord(c->ev_cloud_free, c->stream_slices));
        c->cloud_busy = true;
    }
    for (int i = 0; i < 3; ++i) s.camera_t[i] = c->currentGlobalCamera[i];
    for (int i = 0; i < 9; ++i) s.camera_R[i] = c->rmats.back().m[i];
    s.utime = c->current_utime;
    c->slices.push_back(std::move(s));
    return 0;
}

void drop_slices(kt_ctx* c)
{
    if (c->stream_slices) cudaStreamSynchronize(c->stream_slices);
    c->slices.clear();
    c->slice_arena.rewind();
    c->cloud_busy = false;
}

// Whether the front end builds the depth pyramid, the vertex / normal maps and the colour-integration inputs (which the integration then
// reads): for the ICP modes, and for -r only with the view-angle colour weight (KintinuousTracker.cpp:465, Q10)
bool builds_icp_maps(const kt_config& cfg) { return cfg.odometry == 0 || cfg.odometry == 2 || cfg.angle_color; }

int do_integrate(kt_ctx* c, const M3& Rinv, const V3& t, const int* wrap)
{
    const int rows = c->cfg.rows, cols = c->cfg.cols;
    Intr k = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    IntegrateArgs a;
    a.depth_scaled = c->fe.depth_scaled; a.rows = rows; a.cols = cols; a.k = k; a.volume_size = make_float3(c->size, c->size, c->size);
    a.Rinv = to_mat33(Rinv.m); a.t = make_float3(t.v[0], t.v[1], t.v[2]); a.trunc = c->trunc;
    a.tsdf = c->tsdf; a.color = c->color; a.vol = c->cfg.vol; a.wrap = make_int3(wrap[0], wrap[1], wrap[2]);
    a.rgb = c->in.rgb; a.nmap_curr = c->fe.maps.nmaps[0]; a.angle_color = c->cfg.angle_color != 0;
    for (int k = 0; k < 9; ++k) c->last_int_Rinv[k] = Rinv.m[k];
    for (int k = 0; k < 3; ++k) { c->last_int_t[k] = t.v[k]; c->last_int_wrap[k] = wrap[k]; }
    a.reset_words = c->xwords_dev; a.reset_count = odom_exchange_used(&a.reset_stride); c->xwords_clean = true;       // the prologue launch of integrate() zeroes them
    a.multi = c->world > 1 ? 1 : 0; a.vv = c->vv; a.cw = builds_icp_maps(c->cfg) ? c->fe.cw : 0; a.rgbf = a.cw ? (float4*)c->fe.rgbf : 0;
    return integrate(a, c->ztable, c->stream);
}

// The map pyramids the odometry reads: this frame's vertex / normal maps and the model's prediction from the last frame (volume frame).
struct OdomMaps { const float* const* vmaps_curr; const float* const* nmaps_curr; const float* const* vmaps_g_prev; const float* const* nmaps_g_prev; };

// The odometry kernels' arguments for one pyramid level: the ICP half always, the photometric half (ra) for -r / -ri only.
void odom_level_args(const kt_ctx* c, const OdomMaps& m, int level, IcpLevelArgs* ia, RgbLevelArgs* ra)
{
    const float distThres = 0.10f, angleThres = sinf(20.f * 3.14159254f / 180.f);      // ICPOdometry.h:35-36
    const Intr K = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    const int lr = c->cfg.rows >> level, lc = c->cfg.cols >> level;
    const Intr kl = intr_level(K, level);
    const IcpLevelArgs icp = {m.vmaps_curr[level], m.nmaps_curr[level], m.vmaps_g_prev[level], m.nmaps_g_prev[level], lr, lc, kl, distThres, angleThres};
    *ia = icp;
    if (c->cfg.odometry == 0) return;
    const double SOBEL_SCALE = 1.0 / std::pow(2.0, 3);
    const int minimumGradientMagnitudes[4] = {12, 5, 3, 1};
    const int div = 1 << level;
    ra->dIdx = c->nextdIdx[level]; ra->dIdy = c->nextdIdy[level]; ra->last_depth = c->ph_last.depth[level]; ra->next_depth = c->ph_next.depth[level];
    ra->last_image = c->ph_last.image[level]; ra->next_image = c->ph_next.image[level]; ra->corres = c->corresImg[level]; ra->cloud = c->pointClouds[level];
    ra->rows = lr; ra->cols = lc;
    ra->min_scale = (float)(std::pow((double)minimumGradientMagnitudes[level], 2.0) / std::pow(SOBEL_SCALE, 2.0));
    ra->max_depth_delta = 0.07f; ra->fx = kl.fx; ra->fy = kl.fy; ra->sobel_scale = (float)SOBEL_SCALE;
    // IntrDoublePrecision built from the float Intr (RGBDOdometry.cpp:70-73), per-level division in double
    ra->Kfx = (double)K.fx / div; ra->Kfy = (double)K.fy / div; ra->Kcx = (double)K.cx / div; ra->Kcy = (double)K.cy / div;
}

int run_odometry(kt_ctx* c, const OdomMaps& maps, const M3& Rprev, const V3& tprev, M3* Rcurr, V3* tcurr)
{
    const int mode = c->cfg.odometry;
    int r;
    for (int k = 0; k < 9; ++k) c->pose12_host[k] = Rprev.m[k];
    for (int k = 0; k < 3; ++k) c->pose12_host[9 + k] = tprev.v[k];
    IcpLevelArgs la[LEVELS]; RgbLevelArgs ra[LEVELS];
    for (int level = 0; level < LEVELS; ++level) odom_level_args(c, maps, level, &la[level], &ra[level]);
    int total_iters = 0;
    // KT_FORCE_PER_ITERATION (test hook): take the per-iteration kernels -- the path of images too large for the whole-frame kernels'
    // shared-memory stage -- on an image that would fit, so that it can be compared against the whole-frame path and the reference
    static const bool force_per_iteration = getenv("KT_FORCE_PER_ITERATION") != nullptr;
    bool per_iteration_path = force_per_iteration;
    if (mode == 0 && !force_per_iteration) {
        // ICP-only: the whole coarse-to-fine loop is ONE cooperative launch (kt_icp.cu, icp_frame_kernel)
        for (int level = 0; level < LEVELS; ++level) total_iters += c->iterations[level];
        if (c->timing) cudaEventRecord(c->ev_icp[0], c->stream);
        if (!c->xwords_clean && (r = odom_exchange_reset(c->xwords_dev, c->stream))) return r;
        c->xwords_clean = false;
        ++c->pose_seq;
        unsigned long long* peers[MAX_GPUS];
        for (int g = 0; g < MAX_GPUS; ++g) peers[g] = (unsigned long long*)(c->peer_arena[g] + c->off_xwords);
        if ((r = icp_frame(la, c->iterations, c->pose12_host, c->state, c->xwords_dev, c->trace_dev, &c->state->odo_timeout, c->timing ? c->prof_dev : 0,
                           c->result_dev_alias, c->pose_seq, c->stream, c->split_icp ? peers : 0, c->world, c->rank))) return r;
        if (c->timing) cudaEventRecord(c->ev_icp[1], c->stream);
    } else if (!force_per_iteration) {
        // whole-frame RGB-D / ICP+RGB-D kernel (kt_rgb.cu, rgbd_frame_kernel): ONE cooperative launch for all levels and iterations
        if (!c->xwords_clean && (r = odom_exchange_reset(c->xwords_dev, c->stream))) return r;
        ++c->pose_seq;
        r = rgbd_frame(la, ra, c->iterations, mode == 2 ? 1 : 0, c->pose12_host, c->state, c->xwords_dev, c->trace_dev, &c->state->odo_timeout,
                       c->result_dev_alias, c->pose_seq, c->stream);
        if (r < 0) return r;
        if (r == 0) { c->xwords_clean = false; for (int level = 0; level < LEVELS; ++level) total_iters += c->iterations[level]; }
        else per_iteration_path = true;          // image too large for the shared-memory stage: per-iteration kernels
    }
    if (per_iteration_path) {
        KT_CUDA(cudaMemcpyAsync(c->pose12_dev, c->pose12_host, 12 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        if ((r = odom_begin_frame(c->state, c->pose12_dev, c->stream))) return r;
        for (int level = LEVELS - 1; level >= 0; --level) {
            const RgbLevelArgs& rl = ra[level];
            if (mode != 0 && (r = project_to_point_cloud(c->ph_last.depth[level], c->pointClouds[level], rl.rows, rl.cols, rl.Kfx, rl.Kfy, rl.Kcx, rl.Kcy, c->stream))) return r;
            for (int iter = 0; iter < c->iterations[level]; ++iter) {
                float* trace = (total_iters < MAX_TRACE_ITERS) ? c->trace_dev : 0;
                if (mode == 0) {
                    if ((r = icp_iteration(la[level], c->state, c->partials, trace, 1, c->stream))) return r;
                } else {
                    if ((r = rgb_residual(rl, c->state, c->ipartials, 1, c->stream))) return r;
                    if (mode == 2 && (r = icp_iteration(la[level], c->state, c->partials, 0, 0, c->stream))) return r;
                    if ((r = rgb_iteration(rl, c->state, c->partials, trace, mode == 2 ? 2 : 1, 0.f, c->stream))) return r;
                }
                ++total_iters;
            }
        }
    }
    c->trace_iters = std::min(total_iters, MAX_TRACE_ITERS);
    // one 64-byte read-back of the estimate (+ the trace when someone asked for it later: it stays on the device)
    static_assert(offsetof(OdomState, odo_timeout) == offsetof(OdomState, Rcurr) + 12 * sizeof(float), "the time-out flag travels with the pose");
    bool got = false;
    if (!per_iteration_path && !c->timing) {
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
        std::swap(c->ph_last, c->ph_next);                                                                                                  // RGBDOdometry.cpp:377-381
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

// The front end's arguments for the photometric set alone -- the pyramids and gradients of -r / -ri (RGBDOdometry::populateRGBDData /
// firstRun + computeDerivativeImages, RGBDOdometry.cpp:140-175) into `ph` -- with no depth pyramid, maps or colour inputs.
FrontendArgs photometric_frontend(const kt_ctx* c, const uint16_t* depth_raw, const uint8_t* rgb, const PhotometricPyramid* ph)
{
    FrontendArgs fa; std::memset(&fa, 0, sizeof(fa));
    const Intr K = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    fa.depth_raw = depth_raw; fa.rgb = rgb; fa.rows = c->cfg.rows; fa.cols = c->cfg.cols; fa.k = K; fa.depths = c->fe.maps.depths;
    fa.cut_off = (int)(6.0 * 1000);                                                      // RGBDOdometry.cpp:147
    fa.depth_m = ph ? ph->depth : 0; fa.intensity = ph ? ph->image : 0; fa.dIdx = ph ? c->nextdIdx : 0; fa.dIdy = ph ? c->nextdIdy : 0;
    return fa;
}

// Pose-independent front end of one frame in TWO launches (kt_frontend.cu): bilateral filter + scaleDepth, then the depth pyramid, the
// vertex / normal maps of all levels, the colour-integration inputs and -- for -r / -ri -- the photometric set `ph`.  stale: the previous
// frame's maps when `out` is the spare set (Q7), else null.  Raw frame pointers: the OdometryProvider entry points pass their caller's.
int build_frontend(kt_ctx* c, const uint16_t* depth_raw, const uint8_t* rgb, FrontEnd& out, const MapPyramid* stale, const PhotometricPyramid* ph, cudaStream_t s)
{
    int r;
    const bool icp_maps = builds_icp_maps(c->cfg);
    FrontendArgs fa = photometric_frontend(c, depth_raw, rgb, ph);
    if ((r = bilateral_scale(depth_raw, icp_maps ? out.maps.depths[0] : 0, out.depth_scaled, fa.rows, fa.cols, fa.k, c->cfg.angle_color != 0, s))) return r;
    fa.depth_f = icp_maps ? out.maps.depths[0] : 0; fa.depths = out.maps.depths; fa.vmaps = icp_maps ? out.maps.vmaps : 0; fa.nmaps = icp_maps ? out.maps.nmaps : 0;
    fa.vstale = stale ? stale->vmaps : 0; fa.nstale = stale ? stale->nmaps : 0;
    fa.cw = icp_maps ? out.cw : 0; fa.rgbf = icp_maps ? (float4*)out.rgbf : 0; fa.angle_color = c->cfg.angle_color != 0;
    if (icp_maps || ph) { if ((r = frontend_pyramid(fa, s))) return r; }
    return 0;
}

// densePoseGraph.push_back(DensePose(current_utime, [Rcurr | currentGlobalCamera], isLoopPose)); latestDensePoseId++ and, for tracked
// frames, outputPose (KintinuousTracker.cpp:529-536, :901-914)
void record_dense_pose(kt_ctx* c, bool first, bool keyframe)
{
    kt_dense_pose d;
    d.timestamp = c->current_utime; d.is_loop_pose = (first || keyframe) ? 1 : 0;
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

// The keyframe rule (kt_place.hpp) and, for a keyframe, its capture on the place stream: raw depth and colour copied (the compute stream
// waits for the copy before the inputs can be reused), SURF, the keypoints' 3-D points, the feature count into pinned memory.
int place_capture(kt_ctx* c, bool first, bool* keyframe)
{
    *keyframe = false;
    PlaceStore* ps = c->place.get();
    if (!ps) return 0;
    const float* R = c->rmats.back().m;
    const bool kf = first || ps->times.empty() || c->shifted_last > 0 || place_is_keyframe(R, ps->lastR, c->currentGlobalCamera, ps->lastG);
    if (!kf) return 0;
    for (int k = 0; k < 9; ++k) ps->lastR[k] = R[k];
    for (int k = 0; k < 3; ++k) ps->lastG[k] = c->currentGlobalCamera[k];
    if ((int)ps->times.size() >= ps->maxK) { ps->full = true; return 0; }
    const size_t P = (size_t)ps->rows * ps->cols, k = ps->times.size();
    const Intr K = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    KT_CUDA(cudaStreamWaitEvent(ps->stream, ps->ev_input, 0));
    KT_CUDA(cudaMemcpyAsync(ps->depth + k * P, c->in.depth, P * 2, cudaMemcpyDeviceToDevice, ps->stream));
    KT_CUDA(cudaMemcpyAsync(ps->rgb, c->in.rgb, P * 3, cudaMemcpyDeviceToDevice, ps->stream));
    KT_CUDA(cudaEventRecord(ps->ev_copied, ps->stream));
    KT_CUDA(cudaStreamWaitEvent(c->stream, ps->ev_copied, 0));
    float* kp = ps->kp + k * ps->maxF * 6;
    int r;
    if ((r = surf(ps->rgb, ps->rows, ps->cols, 400.f, ps->maxF, kp, ps->desc + k * ps->maxF * 64, ps->nfeat_dev + k, &ps->surf_ws, ps->stream))) return r;
    if ((r = keypoints_3d(kp, ps->nfeat_dev + k, ps->maxF, ps->depth + k * P, ps->rows, ps->cols, K, ps->xyz + k * ps->maxF * 3, ps->stream))) return r;
    KT_CUDA(cudaMemcpyAsync(ps->nfeat_host + k, ps->nfeat_dev + k, sizeof(int), cudaMemcpyDeviceToHost, ps->stream));
    ps->times.push_back(c->current_utime); ps->dense_idx.push_back((int)c->dense_poses.size());
    *keyframe = true;
    return 0;
}

void mark(kt_ctx* c, int i) { if (c->timing) cudaEventRecord(c->ev[i], c->stream); }

// One axis of the volume shift (.cpp x :675-723, y :729-777, z :783-831): the slab that leaves is cut, its storage planes are stored in
// the map volume, cleared and restored from it, the volume moves n voxels, and the slab is recorded as a slice.
int shift_axis(kt_ctx* c, int axis, int n, int thresh, V3* tcurr)
{
    const int V = c->cfg.vol;
    int lo[3], hi[3];
    const int dir = shift_box(axis, n, thresh, c->overlap, V, lo, hi);                  // kt_shift.hpp: which slab leaves the volume
    if (!dir) return 0;
    int r;
    if ((r = cut_box(c, lo, hi))) return r;
    if ((r = mg_barrier(c))) return r;                                  // peers may still read my boundary plane for their extraction
    int first, planes;                                                  // the storage planes the clear zeroes
    clear_range(axis, dir < 0 ? 1 : 0, V, c->voxelWrap[axis], c->voxelWrap[axis] + n, &first, &planes);
    if (c->mapvol && (r = mapvol_store(c->mapvol.get(), c->tsdf, c->color, V, c->voxelWrap, axis, first, planes, c->stream))) return r;
    if ((r = clear_volume_shared(axis, c->vv, V, first, planes, c->stream))) return r;
    if (c->mapvol && c->mapvol_restore) {                               // give the cleared planes back what the store holds for them
        int after[3] = {c->voxelWrap[0], c->voxelWrap[1], c->voxelWrap[2]};
        after[axis] += n;
        if ((r = mapvol_restore(c->mapvol.get(), c->tsdf, c->color, V, after, axis, first, planes, c->stream))) return r;
    }
    const float step = c->voxel * n;
    c->tvecs.back().v[axis] -= step;
    tcurr->v[axis] -= step;
    c->voxelWrap[axis] += n;
    ++c->shifted_last;
    int vt[3] = {0, 0, 0}; vt[axis] = n;
    return push_slice(c, slice_dimension(vt));                          // mutexOutCloudBuffer (.cpp:1156-1208), with the camera of this frame
}

int process_frame_device(kt_ctx* c, uint64_t utime, kt_pose* out)
{
    const int rows = c->cfg.rows, cols = c->cfg.cols, V = c->cfg.vol;
    const int mode = c->cfg.odometry;
    int r;
    c->shifted_last = 0;
    if (c->place) KT_CUDA(cudaEventRecord(c->place->ev_input, c->stream));       // this frame's raw inputs are in place
    mark(c, 0);
    if (!c->frontend_ready) {
        // the first frame's photometric pyramids are the "last" set (RGBDOdometry::firstRun), every later frame's the "next" set
        const PhotometricPyramid* ph = mode == 0 ? 0 : c->global_time == 0 ? &c->ph_last : &c->ph_next;
        if ((r = build_frontend(c, c->in.depth, c->in.rgb, c->fe, 0, ph, c->stream))) return r;
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
        for (int i = 0; i < LEVELS; ++i) { tl[i].vs = c->fe.maps.vmaps[i]; tl[i].ns = c->fe.maps.nmaps[i]; tl[i].vd = c->vmaps_g_prev[i]; tl[i].nd = c->nmaps_g_prev[i]; tl[i].rows = rows >> i; tl[i].cols = cols >> i; }
        if ((r = transform_maps_pyramid(tl, LEVELS, to_mat33(Rcam.m), make_float3(tcam.v[0], tcam.v[1], tcam.v[2]), c->stream))) return r;
        mark(c, 5);
        ++c->global_time;
        c->current_utime = utime;
        bool kf = false;
        if ((r = place_capture(c, true, &kf))) return r;
        record_dense_pose(c, true, kf);                                                  // .cpp:529-536 (no outputPose on the first frame)
        if (out) kt_get_pose(c, out);
        return 0;
    }

    M3 Rprev = c->rmats.back(); V3 tprev = c->tvecs.back();
    M3 Rcurr = Rprev; V3 tcurr = tprev;
    const OdomMaps maps = {c->fe.maps.vmaps, c->fe.maps.nmaps, c->vmaps_g_prev, c->nmaps_g_prev};
    if ((r = run_odometry(c, maps, Rprev, tprev, &Rcurr, &tcurr))) return r;
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
    for (int axis = 0; axis < 3; ++axis)
        if ((r = shift_axis(c, axis, trans[axis], thresh, &tcurr))) return r;
    int vWrapCopy[3]; vwrap_copy(c, vWrapCopy);
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
    bool kf = false;
    if ((r = place_capture(c, false, &kf))) return r;                                   // .cpp:605-624, 706-718
    record_dense_pose(c, false, kf);                                                     // .cpp:901-914
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
    int r0;
    c->global_time = 0;
    c->rmats.clear(); c->tvecs.clear();
    c->rmats.push_back(m3_identity());
    V3 tb = {{c->volumeBasis[0], c->volumeBasis[1], c->volumeBasis[2]}};
    c->tvecs.push_back(tb);
    for (int i = 0; i < 3; ++i) { c->voxelWrap[i] = 0; c->currentGlobalCamera[i] = c->volumeBasis[i] - c->size * 0.5f; }
    drop_slices(c);
    c->deformed.clear();
    c->deform_arena.rewind();
    c->loops.clear(); c->pgo_nodes.clear();
    std::memset(&c->map_corr, 0, sizeof(c->map_corr));
    if (c->place) {                              // reset(): the place-recognition buffer starts again (.cpp:290-298)
        cudaStreamSynchronize(c->place->stream);
        c->place->times.clear(); c->place->dense_idx.clear(); c->place->processed = 0; c->place->full = false; c->place->last_loop = 0;
        c->place->in_new.clear(); c->place->in_old.clear();
    }
    c->dense_poses.clear();                      // reset(): densePoseGraph.clear(), latestDensePoseId = 0 (.cpp:300-301)
    if (c->mapvol && (r0 = mapvol_empty(c->mapvol.get(), c->stream))) return r0;
    c->trace_iters = 0; c->shifted_last = 0; c->cloud_count = 0;
    c->pf_valid = false; c->pf_built = false; c->frontend_ready = false; c->maps_on_stream = false;
    if (c->stream_copy) cudaStreamSynchronize(c->stream_copy);
    if (c->mg_error_host) { KT_CUDA(cudaStreamSynchronize(c->stream)); *c->mg_error_host = 0; }      // a timed-out cross-GPU barrier is not sticky across resets
    int r = init_shared(c->vv, c->cfg.vol, c->stream);
    if (r) return r;
    // Q7: stale y/z planes of invalid pixels start from a defined state (zeros)
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    for (int l = 0; l < LEVELS; ++l)
        for (float* m : {c->vmaps_g_prev[l], c->nmaps_g_prev[l], c->fe.maps.vmaps[l], c->fe.maps.nmaps[l], c->fe_spare.maps.vmaps[l], c->fe_spare.maps.nmaps[l]})
            KT_CUDA(cudaMemsetAsync(m, 0, (P >> (2 * l)) * 12, c->stream));
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
    std::unique_ptr<kt_ctx> owner(new kt_ctx());
    kt_ctx* c = owner.get();
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
        // KT_ODOM_ITERATIONS=i0,i1,i2,i3 (test hook, finest level first): another schedule.  With one iteration on one level and none
        // elsewhere, the tracked frame's normal equations are those of that level at the previous pose, which a reference can rebuild.
        // Read at every create, so that one process can make trackers with different schedules.
        if (const char* e = getenv("KT_ODOM_ITERATIONS")) {
            int v[4];
            if (sscanf(e, "%d,%d,%d,%d", &v[0], &v[1], &v[2], &v[3]) != 4 || v[0] < 0 || v[1] < 0 || v[2] < 0 || v[3] < 0) {
                set_error("kt_create: KT_ODOM_ITERATIONS must be four non-negative integers i0,i1,i2,i3"); return KT_ERR_INVALID; }
            for (int i = 0; i < 4; ++i) c->iterations[i] = v[i];
        }
    }
    const char* W = "kt_create";
    auto dev = [&](auto** p, size_t n) { return c->mem.device(p, n, W); };
    auto event = [&](cudaEvent_t* e, unsigned int flags) { return c->mem.event(e, flags, W); };
    if (c->mem.stream(&c->stream, W)) return KT_ERR_CUDA;
    const size_t P = (size_t)cfg->rows * cfg->cols;
    {   // shared arena: local volume slab, model maps, raycast colour, barrier flags -- one allocation, one IPC handle
        c->world = cfg->world > 1 ? cfg->world : 1; c->rank = cfg->world > 1 ? cfg->rank : 0;
        c->local_planes = cfg->vol / c->world;
        // colour planes are dealt to the ranks in blocks of mg_block = max(8, V / 64) storage planes (a power of two): small enough
        // that any viewing frustum spreads evenly over the ranks (the frustum's cross-section grows with depth: with V / 16-plane blocks
        // the farthest block alone would hold a third of the work), large enough to amortise the per-column set-up of integrate_kernel,
        // which walks one ownership block per CTA
        c->mg_block = cfg->vol / 64 > 8 ? cfg->vol / 64 : 8;
        { int b = 1; while (b * 2 <= c->mg_block) b *= 2; c->mg_block = b; }
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
        if (dev(&c->arena, off)) return KT_ERR_CUDA;
        KT_CUDA(cudaMemset(c->arena + c->off_flags, 0, 256));
        c->xwords_dev = (unsigned long long*)(c->arena + c->off_xwords);
        KT_CUDA(cudaMemset(c->xwords_dev, 0, odom_exchange_words() * sizeof(unsigned long long))); c->xwords_clean = true;
        c->split_icp = c->world > 1 && getenv("KT_MG_SPLIT_ICP") != nullptr;
        c->tsdf = (int16_t*)(c->arena + c->off_tsdf); c->color = c->arena + c->off_color;
        for (int g = 0; g < MAX_GPUS; ++g) c->peer_arena[g] = c->arena;
        c->connected = (c->world == 1);
        c->epoch = 0;
        c->vv = single_volume(c->tsdf, c->color, cfg->vol);
        c->vv.world = c->world; c->vv.rank = c->rank;
        c->vv.bshift = 0; { int t = c->mg_block; while (t > 1) { t >>= 1; ++c->vv.bshift; } }
        c->vv.nshift = 0; { int t = c->world; while (t > 1) { t >>= 1; ++c->vv.nshift; } }
        if (dev(&c->peer_flags_dev, (size_t)MAX_GPUS)) return KT_ERR_CUDA;
        // the barrier's time-out flag lives in MAPPED host memory: the kernel writes it in place, the host reads it with the pose (no copy)
        if (c->mem.mapped(&c->mg_error_host, 1, W)) return KT_ERR_CUDA; *c->mg_error_host = 0;
        KT_CUDA(cudaHostGetDevicePointer((void**)&c->mg_error_dev, c->mg_error_host, 0));
    }
    if (c->in.alloc(c->mem, P, W) || c->in_spare.alloc(c->mem, P, W) || c->fe.alloc(c->mem, P, W) || c->fe_spare.alloc(c->mem, P, W)) return KT_ERR_CUDA;
    if (cfg->odometry != 0 && (c->ph_last.alloc(c->mem, P, W) || c->ph_next.alloc(c->mem, P, W))) return KT_ERR_CUDA;
    if (c->mem.stream(&c->stream_copy, W)) return KT_ERR_CUDA;
    if (event(&c->ev_prefetch, cudaEventDisableTiming)) return KT_ERR_CUDA;
    for (int i = 0; i < 2; ++i) if (event(&c->ev_done[i], cudaEventDisableTiming)) return KT_ERR_CUDA;
    if (event(&c->ev_maps, cudaEventDisableTiming)) return KT_ERR_CUDA; c->maps_on_stream = false;
    c->last_parity = 0;
    for (int l = 0; l < LEVELS; ++l) {
        size_t Pl = P >> (2 * l);
        c->vmaps_g_prev[l] = (float*)(c->arena + c->off_vmap[l]); c->nmaps_g_prev[l] = (float*)(c->arena + c->off_nmap[l]);
        if (cfg->odometry != 0) {
            if (dev(&c->nextdIdx[l], Pl) || dev(&c->nextdIdy[l], Pl)) return KT_ERR_CUDA;
            if (dev(&c->pointClouds[l], Pl * 3)) return KT_ERR_CUDA;
            uint8_t* ci = 0; if (dev(&ci, Pl * 16)) return KT_ERR_CUDA; c->corresImg[l] = ci;
        }
    }
    c->vmap_curr_color = c->arena + c->off_vcol; if (dev(&c->ztable, (size_t)2 * cfg->vol)) return KT_ERR_CUDA;

    if (dev(&c->state, 1) || dev(&c->partials, (size_t)MAX_PARTIALS * 32)) return KT_ERR_CUDA;
    KT_CUDA(cudaMemset(c->partials, 0, (size_t)MAX_PARTIALS * 32 * sizeof(float)));   // tags start at 0
    if (dev(&c->prof_dev, 64 * 8) || dev(&c->ipartials, (size_t)MAX_PARTIALS * 2)) return KT_ERR_CUDA;
    if (dev(&c->trace_dev, (size_t)MAX_TRACE_ITERS * TRACE_STRIDE) || dev(&c->pose12_dev, 12)) return KT_ERR_CUDA;
    c->cloud_capacity = (size_t)c->cfg.cloud_capacity;
    if (dev(&c->cloud_dev, c->cloud_capacity) || dev(&c->counter_dev, 1)) return KT_ERR_CUDA;
    c->mesh_weight_cull = 8;                                   // -cw default, also the live mesh's until kt_set_slice_meshing
    if (!c->slice_arena.alloc(256)) return KT_ERR_CUDA;      // the first 64 MB slab now, not inside the first shift frame
    c->slice_arena.rewind();
    if (c->mem.stream(&c->stream_slices, W)) return KT_ERR_CUDA;
    if (event(&c->ev_cloud_ready, cudaEventDisableTiming)) return KT_ERR_CUDA;
    if (event(&c->ev_cloud_free, cudaEventDisableTiming)) return KT_ERR_CUDA;
    if (c->mem.pinned(&c->pose12_host, 12, W)) return KT_ERR_CUDA;
    if (c->mem.mapped(&c->result_host, 1, W)) return KT_ERR_CUDA;
    std::memset(c->result_host, 0, sizeof(OdomResult));
    { void* dp = 0; KT_CUDA(cudaHostGetDevicePointer(&dp, c->result_host, 0)); c->result_dev_alias = (float*)dp; }
    c->pose_seq = 0;
    if (c->mem.pinned(&c->trace_host, (size_t)MAX_TRACE_ITERS * TRACE_STRIDE, W)) return KT_ERR_CUDA;
    if (c->mem.pinned(&c->counter_host, 1, W)) return KT_ERR_CUDA;
    for (int i = 0; i < 6; ++i) if (event(&c->ev[i], cudaEventDefault)) return KT_ERR_CUDA;
    for (int i = 0; i < 2; ++i) if (event(&c->ev_icp[i], cudaEventDefault)) return KT_ERR_CUDA;
    for (int i = 0; i < 4; ++i) if (event(&c->ev_krn[i], cudaEventDefault)) return KT_ERR_CUDA;
    for (int i = 0; i < 2; ++i) if (event(&c->ev_span[i], cudaEventDefault)) return KT_ERR_CUDA;
    int r = kt_reset(c); if (r) return r;
    *out = owner.release();
    return KT_OK;
}

int kt_destroy(kt_ctx* c)
{
    delete c;
    return KT_OK;
}

// If (depth, rgb) is the frame kt_prefetch_frame was given, make the prefetched buffer sets the current ones.
static bool adopt_prefetched(kt_ctx* c, const void* depth, const void* rgb)
{
    const bool hit = c->pf_valid && c->pf_depth == depth && c->pf_rgb == rgb;
    if (hit) {
        std::swap(c->in, c->in_spare);
        // a hint before the first frame copies the inputs only: that frame's front end is built on the compute stream into the current set
        if (c->pf_built) { std::swap(c->fe, c->fe_spare); c->frontend_ready = true; }
    }
    // the compute stream waits for the prefetch -- a dropped stale hint's too: its front end may still be writing the photometric "next"
    // buffers this frame is about to rebuild
    if (c->pf_valid) cudaStreamWaitEvent(c->stream, c->ev_prefetch, 0);
    c->pf_valid = false; c->pf_built = false;
    return hit;
}

// kt_process_frame (host buffers) and kt_process_frame_device: the prefetched set, or the frame copied into the current inputs
static int process_frame(kt_ctx* c, const void* depth, const void* rgb, cudaMemcpyKind kind, uint64_t utime, kt_pose* out, const char* who)
{
    if (!c || !depth || !rgb) { set_error("%s: null argument", who); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    if (!adopt_prefetched(c, depth, rgb)) {
        KT_CUDA(cudaMemcpyAsync(c->in.depth, depth, P * 2, kind, c->stream));   // TrackerInterface.cpp:90
        KT_CUDA(cudaMemcpyAsync(c->in.rgb, rgb, P * 3, kind, c->stream));       // TrackerInterface.cpp:91
    }
    const int r = process_frame_device(c, utime, out);
    c->frontend_ready = false;
    c->last_parity ^= 1;
    cudaEventRecord(c->ev_done[c->last_parity], c->stream);      // completion of this frame's last kernel
    return r;
}

int kt_process_frame_device(kt_ctx* c, const uint16_t* depth_dev, const uint8_t* rgb_dev, uint64_t utime, kt_pose* out)
{
    return process_frame(c, depth_dev, rgb_dev, cudaMemcpyDeviceToDevice, utime, out, "kt_process_frame_device");
}

int kt_process_frame(kt_ctx* c, const uint16_t* depth_host, const uint8_t* rgb_host, uint64_t utime, kt_pose* out)
{
    return process_frame(c, depth_host, rgb_host, cudaMemcpyHostToDevice, utime, out, "kt_process_frame");
}

int kt_prefetch_frame(kt_ctx* c, const uint16_t* depth, const uint8_t* rgb)
{
    if (!c || !depth || !rgb) { set_error("kt_prefetch_frame: null argument"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const size_t P = (size_t)c->cfg.rows * c->cfg.cols;
    // the spare set was last read by the frame BEFORE the last one; wait for that frame's completion event only, so the copy and the
    // front end overlap the last frame's integrate / ray-cast.  Host (pinned) or device pointers.
    KT_CUDA(cudaStreamWaitEvent(c->stream_copy, c->ev_done[c->last_parity ^ 1], 0));
    KT_CUDA(cudaMemcpyAsync(c->in_spare.depth, depth, P * 2, cudaMemcpyDefault, c->stream_copy));
    KT_CUDA(cudaMemcpyAsync(c->in_spare.rgb, rgb, P * 3, cudaMemcpyDefault, c->stream_copy));
    c->pf_built = false;
    if (c->global_time > 0) {
        // invalid pixels keep the y/z planes of the previous frame's maps = the set that is current now (Q7); if that set was built on the
        // compute stream (frame not prefetched, e.g. frame 0), wait for its front end -- not for the whole frame
        if (c->maps_on_stream) KT_CUDA(cudaStreamWaitEvent(c->stream_copy, c->ev_maps, 0));
        // photometric odometry: its "next" pyramids were swapped to "last" when the previous frame's odometry finished, so the
        // buffers now called next are free until the coming frame
        int r = build_frontend(c, c->in_spare.depth, c->in_spare.rgb, c->fe_spare, &c->fe.maps, c->cfg.odometry != 0 ? &c->ph_next : 0, c->stream_copy);
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
    const int V = c->cfg.vol;
    int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
    int r = cut_box(c, lo, hi);
    return r ? r : push_slice(c, 7);     // CloudSlice::FINAL
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
        KT_CUDA(cudaEventSynchronize(s.ready.get()));                  // the asynchronous download of this slice has landed
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
        KT_CUDA(cudaEventSynchronize(s.ready.get()));
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
    if (nv || nt) KT_CUDA(cudaEventSynchronize(s.ready.get()));
    if (nv) std::memcpy(verts, s.mesh_verts, nv * sizeof(kt_mesh_vertex));
    if (nt) std::memcpy(tris, s.mesh_tris, nt * 3 * sizeof(uint32_t));
    return KT_OK;
}

// the expanded keys of slice s: up to max_verts vertex edges and max_tris triangle cells (4 x int32 each)
static void slice_mesh_keys(const SliceRec& s, int32_t* vert_edges, size_t max_verts, int32_t* tri_cells, size_t max_tris)
{
    const size_t nv = vert_edges ? std::min(max_verts, s.mesh_nv) : 0, nt = tri_cells ? std::min(max_tris, s.mesh_nt) : 0;
    for (size_t i = 0; i < nv; ++i) mesh_key_global(s.mesh_frame, s.mesh_vkeys[i] / 3, (int)(s.mesh_vkeys[i] % 3), vert_edges + 4 * i);
    for (size_t i = 0; i < nt; ++i) mesh_key_global(s.mesh_frame, s.mesh_tcells[i], 0, tri_cells + 4 * i);
}

int kt_get_slice_mesh_keys(kt_ctx* c, int idx, int32_t* vert_edges, size_t max_verts, int32_t* tri_cells, size_t max_tris)
{
    if (!c || idx < 0 || idx >= (int)c->slices.size()) { set_error("kt_get_slice_mesh_keys: bad index"); return KT_ERR_INVALID; }
    const SliceRec& s = c->slices[idx];
    if (!s.has_mesh) { set_error("kt_get_slice_mesh_keys: slice %d was recorded with meshing off (kt_set_slice_meshing)", idx); return KT_ERR_STATE; }
    if (s.mesh_nv) KT_CUDA(cudaEventSynchronize(s.ready.get()));
    slice_mesh_keys(s, vert_edges, max_verts, tri_cells, max_tris);
    return KT_OK;
}

int kt_get_live_mesh(kt_ctx* c, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris, size_t* n_verts, size_t* n_tris)
{
    if (!c) return KT_ERR_INVALID;
    if (c->world > 1) { set_error("kt_get_live_mesh: a volume shared by %d GPUs cannot be meshed", c->world); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    const int V = c->cfg.vol;
    int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
    int r;
    if ((r = wait_slice_download(c)) || (r = mesh_box(c, lo, hi, false))) return r;
    if (n_verts) *n_verts = c->mesh_nv;
    if (n_tris) *n_tris = c->mesh_nt;
    const size_t nv = verts ? std::min(max_verts, c->mesh_nv) : 0, nt = tris ? std::min(max_tris, c->mesh_nt) : 0;
    if (nv) KT_CUDA(cudaMemcpyAsync(verts, c->mesh_verts.get(), nv * sizeof(kt_mesh_vertex), cudaMemcpyDeviceToHost, c->stream));
    if (nt) KT_CUDA(cudaMemcpyAsync(tris, c->mesh_tris.get(), nt * 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    KT_CUDA(cudaStreamSynchronize(c->stream));
    return KT_OK;
}

// A mesh as parts written back to back: every part's vertices, then every part's triangles with the part's vertices' offset added
struct PlyPart { const kt_mesh_vertex* v; size_t nv; const uint32_t* t; size_t nt; };

// One binary little-endian PLY (vertex: float x y z nx ny nz, uchar red green blue; face: list uchar int vertex_indices)
static int write_mesh_ply(const char* path, const std::vector<PlyPart>& parts, const char* who)
{
    size_t nv = 0, nt = 0;
    for (const PlyPart& p : parts) { nv += p.nv; nt += p.nt; }
    if (nv > 0x7fffffffu) { set_error("%s: %zu vertices do not fit the PLY's int indices", who, nv); return KT_ERR_CAPACITY; }
    FILE* f = fopen(path, "wb");
    if (!f) { set_error("%s: cannot open %s", who, path); return KT_ERR_INVALID; }
    fprintf(f, "ply\nformat binary_little_endian 1.0\nelement vertex %zu\nproperty float x\nproperty float y\nproperty float z\n"
               "property float nx\nproperty float ny\nproperty float nz\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n"
               "element face %zu\nproperty list uchar int vertex_indices\nend_header\n", nv, nt);
    std::vector<unsigned char> buf;
    bool ok = true;
    for (const PlyPart& p : parts) {                              // x86 / aarch64 hosts are little-endian: records are the raw bytes
        if (!p.nv) continue;
        buf.resize(p.nv * 27);
        for (size_t i = 0; i < p.nv; ++i) {
            std::memcpy(&buf[i * 27], &p.v[i].x, 24);
            buf[i * 27 + 24] = p.v[i].r; buf[i * 27 + 25] = p.v[i].g; buf[i * 27 + 26] = p.v[i].b;
        }
        ok = ok && fwrite(buf.data(), 1, buf.size(), f) == buf.size();
    }
    uint32_t base = 0;
    for (const PlyPart& p : parts) {
        if (!ok) break;
        buf.resize(p.nt * 13);
        for (size_t t = 0; t < p.nt; ++t) {
            buf[t * 13] = 3;
            for (int k = 0; k < 3; ++k) { const int32_t v = (int32_t)(p.t[3 * t + k] + base); std::memcpy(&buf[t * 13 + 1 + 4 * k], &v, 4); }
        }
        ok = ok && fwrite(buf.data(), 1, buf.size(), f) == buf.size();
        base += (uint32_t)p.nv;
    }
    if (fclose(f) != 0) ok = false;
    if (!ok) { set_error("%s: writing %s failed", who, path); return KT_ERR_CUDA; }
    return KT_OK;
}

// The meshes of the first n_slices slices as one binary PLY; with `deformed`, the vertices of the last kt_deform_map
static int save_mesh_ply(kt_ctx* c, const char* path, size_t n_slices, bool deformed, const char* who)
{
    bool any = false;
    for (size_t i = 0; i < n_slices; ++i) if (c->slices[i].has_mesh) any = true;
    if (!any) { set_error("%s: no slice was recorded with meshing on (kt_set_slice_meshing)", who); return KT_ERR_STATE; }
    std::vector<PlyPart> parts;
    for (size_t k = 0; k < n_slices; ++k) {
        const auto& s = c->slices[k];
        if (!s.has_mesh) continue;
        if (s.mesh_nv) KT_CUDA(cudaEventSynchronize(s.ready.get()));
        parts.push_back(PlyPart{deformed ? c->deformed[k].mesh_verts : s.mesh_verts, s.mesh_nv, s.mesh_tris, s.mesh_nt});
    }
    return write_mesh_ply(path, parts, who);
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
    // the scratch below is freed after the tracker stream has finished with it; c->deformed is left empty on an error
    c->deformed.clear();
    cudaStream_t s = c->stream;
    Allocations mem(s); const char* W = "kt_deform_map scratch";
    float* d_npos; uint64_t* d_ntime; double* d_x; uint64_t* d_t; int32_t* d_ids; double* d_w; unsigned char* d_in; unsigned char* d_out;
    if (mem.device(&d_npos, npos.size(), W) || mem.device(&d_ntime, ntime.size(), W) || mem.device(&d_x, (size_t)nn * 12, W) ||
        mem.device(&d_t, nmax, W) || mem.device(&d_ids, nmax * 4, W) || mem.device(&d_w, nmax * 4, W) || mem.device(&d_in, nmax * sizeof(kt_point_xyzrgbnormal), W)) return KT_ERR_CUDA;
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
    std::vector<kt_ctx::Deformed> def(c->slices.size());
    for (size_t i = 0; i < c->slices.size(); ++i) { def[i].processed = c->slices[i].processed; def[i].mesh_verts = c->slices[i].mesh_verts; }
    if (!report->deformed) { c->deformed = std::move(def); return 0; }               // the map as recorded
    c->deform_arena.rewind();
    if (mem.device(&d_out, nmax * sizeof(kt_point_xyzrgbnormal), W)) return KT_ERR_CUDA;
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
            void* h = c->deform_arena.alloc(cnt * rec);
            if (!h) { set_error("kt_deform_map: pinned host memory for %zu deformed records", cnt); return KT_ERR_CUDA; }
            KT_CUDA(cudaMemcpyAsync(h, (const char*)d_out + off * rec, cnt * rec, cudaMemcpyDeviceToHost, s));
            if (kind == 0) def[i].processed = (kt_point_xyzrgbnormal*)h; else def[i].mesh_verts = (kt_mesh_vertex*)h;
            off += cnt;
        }
        KT_CUDA(cudaStreamSynchronize(s));                                            // vt and the device buffers are reused
    }
    c->deformed = std::move(def);
    return 0;
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
    r = deform_run(c, npos, ntime, cons, report);
    if (r) return r;
    // the correction later slices follow: the last corrected pose and the dense pose it corrects (the last one with its timestamp,
    // as iSAM's camera map keeps it); point constraints alone correct no pose
    kt_ctx::MapCorrection mc; std::memset(&mc, 0, sizeof(mc));
    for (int e = 0; e < 4; ++e) mc.tracked[5 * e] = mc.corrected[5 * e] = 1.f;
    if (n) {
        mc.time = corrected[n - 1].timestamp;
        std::memcpy(mc.corrected, corrected[n - 1].pose, sizeof(mc.corrected));
        for (size_t i = nd; i-- > 0;)
            if (c->dense_poses[i].timestamp == mc.time) { std::memcpy(mc.tracked, c->dense_poses[i].pose, sizeof(mc.tracked)); break; }
    }
    c->map_corr = mc;
    return KT_OK;
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
    std::vector<double> X(X0.size());
    kt_pgo_report pr;
    int r;
    {   // the poses on the device, freed after the tracker stream has finished with them
        Allocations mem(c->stream);
        double* d_X;
        if ((r = mem.device(&d_X, X0.size(), "kt_close_loop poses"))) return r;
        KT_CUDA(cudaMemcpyAsync(d_X, X0.data(), X0.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        if ((r = pgo_optimise(d_X, n, f.data(), (int)f.size(), d_X, &pr, c->stream))) return r;
        KT_CUDA(cudaMemcpy(X.data(), d_X, X.size() * sizeof(double), cudaMemcpyDeviceToHost));
    }
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
        c->map_corr.time = nodes[n - 1].timestamp;
        std::memcpy(c->map_corr.tracked, c->dense_poses[take[n - 1]].pose, sizeof(c->map_corr.tracked));
        std::memcpy(c->map_corr.corrected, nodes[n - 1].pose, sizeof(c->map_corr.corrected));
    }
    c->loops.swap(loops);
    c->pgo_nodes.swap(nodes);
    return KT_OK;
}

int kt_num_loops(kt_ctx* c) { return c ? (int)c->loops.size() : 0; }

// ---- loop detection (PlaceRecognition, backend/PlaceRecognition.cpp) ----
int kt_default_loop_detection(kt_loop_detection_params* p)
{
    if (!p) return KT_ERR_INVALID;
    p->enabled = 1; p->inlier_ratio = 0.35f; p->loop_throttle_s = 30.0; p->isam_thresh = 10.0; p->node_spacing = 0.8f; p->pose_spacing = 0.f;
    p->max_keyframes = 1000; p->max_features = 1000; p->exclude_recent = 20; p->close = 1;
    return KT_OK;
}

int kt_set_loop_detection(kt_ctx* c, const kt_loop_detection_params* p)
{
    if (!c) return KT_ERR_INVALID;
    KT_CUDA(cudaSetDevice(c->cfg.device));
    if (!p || !p->enabled) { c->place.reset(); return KT_OK; }
    if (c->world > 1) { set_error("kt_set_loop_detection: a volume shared by %d GPUs has no loop detection", c->world); return KT_ERR_INVALID; }
    if (p->max_keyframes < 1 || p->max_features < 2 || p->exclude_recent < 1 || !(p->inlier_ratio >= 0.f) || !(p->loop_throttle_s >= 0.0)) {
        set_error("kt_set_loop_detection: bad parameters"); return KT_ERR_INVALID;
    }
    if (c->place) {          // new parameters; the store is kept when its shape is unchanged
        if (c->place->maxK == p->max_keyframes && c->place->maxF == p->max_features) { c->place->p = *p; return KT_OK; }
        c->place.reset();
    }
    std::unique_ptr<PlaceStore> ps(new PlaceStore());
    ps->p = *p; ps->rows = c->cfg.rows; ps->cols = c->cfg.cols; ps->maxK = p->max_keyframes; ps->maxF = p->max_features;
    const size_t P = (size_t)ps->rows * ps->cols, K = (size_t)ps->maxK, F = (size_t)ps->maxF;
    const char* W = "the loop detection store";
    auto dev = [&](auto** q, size_t n) { return ps->mem.device(q, n, W); };
    if (ps->mem.stream(&ps->stream, W) || ps->mem.event(&ps->ev_input, cudaEventDisableTiming, W) || ps->mem.event(&ps->ev_copied, cudaEventDisableTiming, W) ||
        ps->mem.pinned(&ps->nfeat_host, K, W)) return KT_ERR_CUDA;
    if (dev(&ps->depth, K * P) || dev(&ps->rgb, P * 3) || dev(&ps->kp, K * F * 6) || dev(&ps->desc, K * F * 64) || dev(&ps->xyz, K * F * 3) || dev(&ps->nfeat_dev, K) ||
        dev(&ps->best, K * F) || dev(&ps->d1, K * F) || dev(&ps->d2, K * F) || dev(&ps->pass, K * F) || dev(&ps->seg_passes, K) ||
        dev(&ps->pn, F * 3) || dev(&ps->po, F * 3) || dev(&ps->uv, F * 2) || dev(&ps->pose, 12) || dev(&ps->inl, F) || dev(&ps->ninl, 1)) return KT_ERR_CUDA;
    for (int s2 = 0; s2 < 2; ++s2) {
        if (ps->maps[s2].alloc(ps->mem, P, W)) return KT_ERR_CUDA;
        for (int l = 0; l < LEVELS; ++l)
            for (float* m : {ps->maps[s2].vmaps[l], ps->maps[s2].nmaps[l]}) KT_CUDA(cudaMemset(m, 0, (P >> (2 * l)) * 12));
        if (dev(&ps->cloud[s2], P) || dev(&ps->cent[s2], P)) return KT_ERR_CUDA;
    }
    if (dev(&ps->d2fit, P + 8) || dev(&ps->state, 1)) return KT_ERR_CUDA;
    KT_CUDA(cudaMemset(ps->state, 0, sizeof(OdomState)));
    if (dev(&ps->xwords, odom_exchange_words()) || dev(&ps->trace, (size_t)MAX_TRACE_ITERS * TRACE_STRIDE)) return KT_ERR_CUDA;
    c->place = std::move(ps);
    return KT_OK;
}

int kt_num_keyframes(kt_ctx* c, int* full)
{
    if (!c) return 0;
    if (full) *full = c->place && c->place->full ? 1 : 0;
    return c->place ? (int)c->place->times.size() : 0;
}

int kt_get_keyframe(kt_ctx* c, int idx, uint64_t* timestamp, int* dense_pose_index, int* n_features)
{
    if (!c || !c->place || idx < 0 || idx >= (int)c->place->times.size()) { set_error("kt_get_keyframe: bad argument"); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    KT_CUDA(cudaStreamSynchronize(c->place->stream));
    if (timestamp) *timestamp = c->place->times[idx];
    if (dense_pose_index) *dense_pose_index = c->place->dense_idx[idx];
    if (n_features) *n_features = c->place->nfeat_host[idx];
    return KT_OK;
}

namespace {

// 4 x 4 row-major FP64 helpers of the detection chain
void m4_from12(const double* p, double* T) { for (int r = 0; r < 3; ++r) { for (int k = 0; k < 3; ++k) T[r * 4 + k] = p[r * 3 + k]; T[r * 4 + 3] = p[9 + r]; } T[12] = T[13] = T[14] = 0; T[15] = 1; }
void m4_mul(const double* A, const double* B, double* C) { for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += A[i * 4 + k] * B[k * 4 + j]; C[i * 4 + j] = s; } }
void m4_rigid_inverse(const double* T, double* I)
{
    for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) I[i * 4 + j] = T[j * 4 + i]; I[i * 4 + 3] = -(T[0 * 4 + i] * T[3] + T[1 * 4 + i] * T[7] + T[2 * 4 + i] * T[11]); }
    I[12] = I[13] = I[14] = 0; I[15] = 1;
}

// One keyframe through the chain (PlaceRecognition::process + processLoopClosureDetection, PlaceRecognition.cpp:51-209).
int place_process(kt_ctx* c, int q, kt_place_result* res)
{
    PlaceStore* ps = c->place.get();
    cudaStream_t s = c->stream;
    const size_t P = (size_t)ps->rows * ps->cols, F = (size_t)ps->maxF;
    const float intr[4] = {c->cfg.fx, c->cfg.fy, c->cfg.cx, c->cfg.cy};
    const Intr K = {intr[0], intr[1], intr[2], intr[3]};
    const float RATIO = 0.49f;
    const int MIN_PASSES = 40, MIN_MATCHES = 40, PNP_ITERS = 500;
    std::memset(res, 0, sizeof(*res));
    res->keyframe = q; res->time = ps->times[q]; res->candidate = -1; res->fitness = -1.0;
    int r;
    if (place_throttled(ps->last_loop, res->time, ps->p.loop_throttle_s)) { res->stage = KT_PLACE_THROTTLED; return 0; }
    res->stage = KT_PLACE_NO_CANDIDATE;
    const int nseg = q - ps->p.exclude_recent + 1;
    if (nseg <= 0) return 0;
    // retrieval: every feature of every keyframe old enough against the new keyframe's
    if ((r = match_ratio(ps->desc, nseg, ps->maxF, ps->nfeat_dev, ps->desc + (size_t)q * F * 64, ps->nfeat_dev + q, ps->maxF, RATIO, ps->best, ps->d1, ps->d2,
                         ps->pass, ps->seg_passes, s))) return r;
    std::vector<int> passes((size_t)q + 1, 0);
    KT_CUDA(cudaMemcpyAsync(passes.data(), ps->seg_passes, (size_t)nseg * sizeof(int), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    const int cand = place_select_candidate(passes.data(), q, ps->p.exclude_recent, MIN_PASSES);
    if (cand < 0) return 0;
    res->candidate = cand; res->candidate_time = ps->times[cand]; res->passes = passes[cand];
    // 3-D matching of the pair in surfMatch3D's order (Surf3DTools.h:105-176): the ratio test over ALL features of the two stored blocks
    // (every old feature against every new one, counts on the device), one match per new feature, then the pairs without a 3-D point
    // dropped (kt_place.hpp place_match_3d)
    const int nq = ps->nfeat_host[q], nc = ps->nfeat_host[cand];
    if ((r = match_ratio(ps->desc + (size_t)cand * F * 64, 1, ps->maxF, ps->nfeat_dev + cand, ps->desc + (size_t)q * F * 64, ps->nfeat_dev + q, ps->maxF, RATIO,
                         ps->best, ps->d1, ps->d2, ps->pass, 0, s))) return r;
    std::vector<float> kq((size_t)nq * 6), kc((size_t)nc * 6), xq((size_t)nq * 3), xc((size_t)nc * 3);
    std::vector<int> best((size_t)nc); std::vector<float> d1((size_t)nc); std::vector<unsigned char> pass((size_t)nc);
    KT_CUDA(cudaMemcpyAsync(kq.data(), ps->kp + (size_t)q * F * 6, kq.size() * 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(kc.data(), ps->kp + (size_t)cand * F * 6, kc.size() * 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(xq.data(), ps->xyz + (size_t)q * F * 3, xq.size() * 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(xc.data(), ps->xyz + (size_t)cand * F * 3, xc.size() * 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(best.data(), ps->best, best.size() * 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(d1.data(), ps->d1, d1.size() * 4, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(pass.data(), ps->pass, pass.size(), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    std::vector<int> oi, ni;
    place_match_3d(best.data(), d1.data(), pass.data(), nc, nq, xc.data(), xq.data(), oi, ni);
    const int m = (int)oi.size();
    res->matches = m; res->stage = KT_PLACE_MATCHES;
    if (m < MIN_MATCHES) return 0;
    // PnP RANSAC: new 3-D points, old keypoints (PNPSolver.cpp:51-75)
    std::vector<float> pn((size_t)m * 3), po((size_t)m * 3), uv((size_t)m * 2), kpn((size_t)m * 2), kpo((size_t)m * 2);
    for (int k = 0; k < m; ++k) {
        const int a = ni[k], b = oi[k];
        for (int e = 0; e < 3; ++e) { pn[(size_t)k * 3 + e] = xq[(size_t)a * 3 + e]; po[(size_t)k * 3 + e] = xc[(size_t)b * 3 + e]; }
        uv[(size_t)k * 2] = kc[(size_t)b * 6]; uv[(size_t)k * 2 + 1] = kc[(size_t)b * 6 + 1];
        kpn[(size_t)k * 2] = kq[(size_t)a * 6]; kpn[(size_t)k * 2 + 1] = kq[(size_t)a * 6 + 1]; kpo[(size_t)k * 2] = uv[(size_t)k * 2]; kpo[(size_t)k * 2 + 1] = uv[(size_t)k * 2 + 1];
    }
    KT_CUDA(cudaMemcpyAsync(ps->pn, pn.data(), pn.size() * 4, cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(ps->po, po.data(), po.size() * 4, cudaMemcpyHostToDevice, s));
    KT_CUDA(cudaMemcpyAsync(ps->uv, uv.data(), uv.size() * 4, cudaMemcpyHostToDevice, s));
    PnpArgs pa; pa.p_new = ps->pn; pa.p_old = ps->po; pa.uv_old = ps->uv; pa.n = m; pa.k = K; pa.iterations = PNP_ITERS; pa.threshold_px = 2.f;
    pa.seed = 0x4b696e74756f7573ull;
    if ((r = pnp_ransac(pa, &ps->pnp_ws, ps->pose, ps->inl, ps->ninl, s))) return r;
    double pose12[12]; int n_in = 0; std::vector<unsigned char> inl((size_t)m);
    KT_CUDA(cudaMemcpyAsync(pose12, ps->pose, sizeof(pose12), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(&n_in, ps->ninl, sizeof(int), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(inl.data(), ps->inl, inl.size(), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    res->inliers = n_in; res->inlier_ratio = (float)n_in / (float)m; res->stage = KT_PLACE_INLIERS;
    if (!((float)n_in / (float)m > ps->p.inlier_ratio)) return 0;
    // dense check: both keyframes' maps by the fused front end, the new one moved into the old camera by the PnP pose, then the tracker's
    // whole-frame projective ICP with the old keyframe's maps as the model (camera at the identity)
    double Tp[16]; m4_from12(pose12, Tp);
    for (int sidx = 0; sidx < 2; ++sidx) {
        const uint16_t* dk = ps->depth + (size_t)(sidx == 0 ? cand : q) * P;
        if ((r = bilateral_scale(dk, ps->maps[sidx].depths[0], 0, ps->rows, ps->cols, K, false, s))) return r;
        FrontendArgs fa; std::memset(&fa, 0, sizeof(fa));
        fa.depth_f = ps->maps[sidx].depths[0]; fa.depth_raw = dk; fa.rows = ps->rows; fa.cols = ps->cols; fa.k = K;
        fa.depths = ps->maps[sidx].depths; fa.vmaps = ps->maps[sidx].vmaps; fa.nmaps = ps->maps[sidx].nmaps;
        if ((r = frontend_pyramid(fa, s))) return r;
    }
    float Rp[9], tp[3];
    for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) Rp[i * 3 + j] = (float)Tp[i * 4 + j]; tp[i] = (float)Tp[i * 4 + 3]; }
    const MapPyramid& mc = ps->maps[1];
    TransformLevel tl[LEVELS];
    for (int l = 0; l < LEVELS; ++l) { tl[l].vs = mc.vmaps[l]; tl[l].ns = mc.nmaps[l]; tl[l].vd = mc.vmaps[l]; tl[l].nd = mc.nmaps[l]; tl[l].rows = ps->rows >> l; tl[l].cols = ps->cols >> l; }
    if ((r = transform_maps_pyramid(tl, LEVELS, to_mat33(Rp), make_float3(tp[0], tp[1], tp[2]), s))) return r;
    const OdomMaps maps = {mc.vmaps, mc.nmaps, ps->maps[0].vmaps, ps->maps[0].nmaps};
    IcpLevelArgs la[LEVELS]; RgbLevelArgs ra[LEVELS];
    for (int l = 0; l < LEVELS; ++l) odom_level_args(c, maps, l, &la[l], &ra[l]);
    const float pose_id[12] = {1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0};
    if ((r = odom_exchange_reset(ps->xwords, s))) return r;
    if ((r = icp_frame(la, c->iterations, pose_id, ps->state, ps->xwords, ps->trace, &ps->state->odo_timeout, 0, 0, 0, s))) return r;
    float Rt[13];
    KT_CUDA(cudaMemcpyAsync(Rt, (char*)ps->state + offsetof(OdomState, Rcurr), 13 * sizeof(float), cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    if (((int*)Rt)[12]) { set_error("kt_detect_loops: the ICP kernel's grid-wide sum gave up"); return KT_ERR_STATE; }
    double dT[16], T[16], C[16];
    for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) dT[i * 4 + j] = Rt[i * 3 + j]; dT[i * 4 + 3] = Rt[9 + i]; }
    dT[12] = dT[13] = dT[14] = 0; dT[15] = 1;
    m4_mul(dT, Tp, T);                 // new camera -> old camera
    m4_rigid_inverse(T, C);            // old -> new: the pose of the old camera in the new one (icpDepthFrames' result)
    // fitness: the old keyframe's cloud moved by C against the new one's, both at 2.5 voxels (PlaceRecognition.cpp:238-276)
    if ((r = depth_to_cloud(ps->depth + (size_t)cand * P, ps->rows, ps->cols, K, ps->cloud[0], s))) return r;
    if ((r = depth_to_cloud(ps->depth + (size_t)q * P, ps->rows, ps->cols, K, ps->cloud[1], s))) return r;
    float T12[12];
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 4; ++j) T12[i * 4 + j] = (float)C[i * 4 + j];
    size_t ns = 0, nd = 0;
    if ((r = cloud_fitness(ps->cloud[0], P, ps->cloud[1], P, 2.5f * c->voxel, T12, &ps->ws[0], &ps->ws[1], ps->cent[0], ps->cent[1], P, ps->d2fit, &res->fitness, &ns, &nd, s))) return r;
    res->stage = KT_PLACE_FITNESS;
    for (int k = 0; k < 16; ++k) res->constraint.constraint[k] = C[k];      // the pose the fitness was measured at, loop or not
    if (!(res->fitness >= 0.0 && res->fitness < 0.01)) return 0;
    // the loop: inliers back-projected at their truncated pixels (DepthCamera::projectInlierMatches)
    std::vector<uint16_t> hd_new(P), hd_old(P);
    KT_CUDA(cudaMemcpyAsync(hd_new.data(), ps->depth + (size_t)q * P, P * 2, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaMemcpyAsync(hd_old.data(), ps->depth + (size_t)cand * P, P * 2, cudaMemcpyDeviceToHost, s));
    KT_CUDA(cudaStreamSynchronize(s));
    ps->in_new.emplace_back(); ps->in_old.emplace_back();
    std::vector<float>& a1 = ps->in_new.back(); std::vector<float>& a2 = ps->in_old.back();
    place_project_inliers(kpn.data(), kpo.data(), inl.data(), m, hd_new.data(), hd_old.data(), ps->rows, ps->cols, intr, a1, a2);
    res->stage = KT_PLACE_LOOP;
    res->constraint.time1 = res->time; res->constraint.time2 = res->candidate_time;
    res->constraint.n_inliers = a1.size() / 3;
    res->constraint.inliers1 = a1.empty() ? 0 : a1.data(); res->constraint.inliers2 = a2.empty() ? 0 : a2.data();
    return 0;
}

} // namespace

int kt_detect_loops(kt_ctx* c, kt_place_result* out, size_t capacity, size_t* n_out)
{
    if (n_out) *n_out = 0;
    if (!c || (!out && capacity)) { set_error("kt_detect_loops: bad argument"); return KT_ERR_INVALID; }
    if (c->world > 1) { set_error("kt_detect_loops: a volume shared by %d GPUs has no loop detection", c->world); return KT_ERR_INVALID; }
    if (!c->place) { set_error("kt_detect_loops: loop detection is off (kt_set_loop_detection)"); return KT_ERR_STATE; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    PlaceStore* ps = c->place.get();
    KT_CUDA(cudaStreamSynchronize(ps->stream));                  // every capture has landed
    ps->in_new.clear(); ps->in_old.clear();
    const size_t pending = ps->times.size() - ps->processed;
    ps->in_new.reserve(std::min(capacity, pending)); ps->in_old.reserve(std::min(capacity, pending));  // constraints point into these until the next call
    size_t n = 0;
    while (n < capacity && ps->processed < ps->times.size()) {
        kt_place_result* res = &out[n];
        int r = place_process(c, (int)ps->processed, res);
        ++ps->processed; ++n;
        if (n_out) *n_out = n;
        if (r) return r;
        if (res->stage == KT_PLACE_LOOP && ps->p.close) {
            r = kt_close_loop(c, &res->constraint, ps->p.pose_spacing, ps->p.node_spacing, ps->p.isam_thresh, &res->report);
            if (r) return r;
            res->closed = res->report.accepted;
        }
        // the -lt throttle starts with a loop the backend ACCEPTS (Deformation.cpp:258-260 sets lastLoopTime after the iSAM gate); with
        // close = 0 the library never learns the outcome, so it starts with every loop found
        if (res->stage == KT_PLACE_LOOP && (!ps->p.close || res->closed)) ps->last_loop = res->time;
    }
    return KT_OK;
}

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

// The correction slices recorded after the last deformation follow: C = P_corr(t) P_tracked(t)^-1 in FP64, the rigid inverse
// [R^T | -R^T t], rounded to float
static RigidF map_correction(const kt_ctx* c)
{
    const float* Pt = c->map_corr.tracked; const float* Pc = c->map_corr.corrected;
    RigidF C;
    for (int a = 0; a < 3; ++a) {
        for (int b = 0; b < 3; ++b) {
            double v = 0;
            for (int k = 0; k < 3; ++k) v += (double)Pc[4 * a + k] * (double)Pt[4 * b + k];
            C.R[3 * a + b] = (float)v;
        }
        double t = Pc[4 * a + 3];
        for (int b = 0; b < 3; ++b) {
            double v = 0;
            for (int k = 0; k < 3; ++k) v += (double)Pc[4 * a + k] * (double)Pt[4 * b + k];
            t -= v * (double)Pt[4 * b + 3];
        }
        C.t[a] = (float)t;
    }
    return C;
}

// The map as one cloud (kt_get_map_cloud, kt_save_map_pcd; the header describes which / dedupe).  The points go to out (up to capacity),
// or, with `grow`, to a host vector sized to the full count.  Device work, if any, runs on the slice stream with scratch that is freed
// before returning; nothing the tracker reads is written.
static int map_cloud(kt_ctx* c, int which, int dedupe, kt_point_xyzrgbnormal* out, size_t capacity, std::vector<kt_point_xyzrgbnormal>* grow,
                     size_t* count, kt_map_report* report, const char* who)
{
    kt_map_report R; std::memset(&R, 0, sizeof(R));
    if (report) *report = R;
    if (count) *count = 0;
    if (which != 0 && which != 1) { set_error("%s: which must be 0 (recorded map) or 1 (corrected map)", who); return KT_ERR_INVALID; }
    if (c->world > 1) { set_error("%s: each of the %d GPUs sharing the volume holds only its own voxels of a slice", who, c->world); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    if (c->stream_slices) KT_CUDA(cudaStreamSynchronize(c->stream_slices));           // every slice has landed in its pinned buffers
    // slices [0, covered) come from the deformed copies; with which = 1 the later ones are moved rigidly and follow them
    const size_t covered = which == 1 ? c->deformed.size() : c->slices.size();
    size_t n = 0, n_fixed = 0;
    for (size_t i = 0; i < c->slices.size(); ++i) {
        const SliceRec& s = c->slices[i];
        if (!s.has_processed) continue;
        ++R.slices; n += s.processed_count;
        if (i < covered) n_fixed += s.processed_count; else ++R.moved_slices;
    }
    if (!R.slices) { set_error("%s: no slice was recorded with slice processing on (kt_set_slice_processing)", who); return KT_ERR_STATE; }
    if (which == 1 && c->deformed.empty()) { set_error("%s: no kt_deform_map / kt_close_loop has deformed the map since the last reset", who); return KT_ERR_STATE; }
    auto src = [&](size_t i) -> const kt_point_xyzrgbnormal* { return which == 1 && i < covered ? c->deformed[i].processed : c->slices[i].processed; };
    const size_t rec = sizeof(kt_point_xyzrgbnormal);
    R.input_points = n;
    if (!dedupe && n_fixed == n) {                                                     // a concatenation of pinned host buffers
        R.output_points = n;
        if (grow) { grow->resize(n); out = grow->data(); capacity = n; }
        size_t off = 0;
        for (size_t i = 0; i < c->slices.size() && out && off < capacity; ++i) {
            const SliceRec& s = c->slices[i];
            if (!s.has_processed || !s.processed_count) continue;
            const size_t k = std::min(s.processed_count, capacity - off);
            std::memcpy(out + off, src(i), k * rec);
            off += k;
        }
    } else if (n) {
        cudaStream_t s = c->stream_slices;
        Allocations mem(s);
        unsigned char* d_in = 0; unsigned char* d_out = 0;
        cudaEvent_t ev[4];
        for (int e = 0; e < 4; ++e) if (mem.event(&ev[e], cudaEventDefault, who)) return KT_ERR_CUDA;
        if (mem.device(&d_in, n * rec, who) || (dedupe && mem.device(&d_out, n * rec, who))) return KT_ERR_CUDA;
        KT_CUDA(cudaEventRecord(ev[0], s));
        size_t off = 0;
        for (size_t i = 0; i < c->slices.size(); ++i) {
            const SliceRec& sl = c->slices[i];
            if (!sl.has_processed || !sl.processed_count) continue;
            KT_CUDA(cudaMemcpyAsync((char*)d_in + off * rec, src(i), sl.processed_count * rec, cudaMemcpyHostToDevice, s));
            off += sl.processed_count;
        }
        KT_CUDA(cudaEventRecord(ev[1], s));
        if (n_fixed < n) { int r = rigid_move((kt_point_xyzrgbnormal*)d_in + n_fixed, n - n_fixed, map_correction(c), s); if (r) return r; }
        size_t m = n;
        float ms2[2] = {0.f, 0.f};
        if (dedupe) { int r = voxel_grid(d_in, n, 1, c->voxel, d_out, n, &m, &R.pcl_would_skip, ms2, s); if (r) return r; }
        R.output_points = m;
        if (grow) { grow->resize(m); out = grow->data(); capacity = m; }
        KT_CUDA(cudaEventRecord(ev[2], s));
        const size_t k = out ? std::min(m, capacity) : 0;
        if (k) KT_CUDA(cudaMemcpyAsync(out, dedupe ? d_out : d_in, k * rec, cudaMemcpyDeviceToHost, s));
        KT_CUDA(cudaEventRecord(ev[3], s));
        KT_CUDA(cudaStreamSynchronize(s));
        KT_CUDA(cudaEventElapsedTime(&R.upload_ms, ev[0], ev[1]));
        KT_CUDA(cudaEventElapsedTime(&R.download_ms, ev[2], ev[3]));
        KT_CUDA(cudaEventElapsedTime(&R.total_ms, ev[0], ev[3]));
        R.sort_ms = ms2[0]; R.centroid_ms = ms2[1];
    }
    if (count) *count = R.output_points;
    if (report) *report = R;
    return KT_OK;
}

int kt_get_map_cloud(kt_ctx* c, int which, int dedupe, kt_point_xyzrgbnormal* out, size_t capacity, size_t* count, kt_map_report* report)
{
    if (!c || !count) { set_error("kt_get_map_cloud: bad argument"); return KT_ERR_INVALID; }
    return map_cloud(c, which, dedupe != 0, out, out ? capacity : 0, 0, count, report, "kt_get_map_cloud");
}

// PCL 1.7.2 PCDWriter::writeBinary of a PointXYZRGBNormal cloud (generateHeader, then the fields packed without padding)
int kt_save_map_pcd(kt_ctx* c, const char* path, int which, int dedupe, kt_map_report* report)
{
    if (!c || !path) { set_error("kt_save_map_pcd: bad argument"); return KT_ERR_INVALID; }
    std::vector<kt_point_xyzrgbnormal> cloud;
    size_t n = 0;
    int r = map_cloud(c, which, dedupe != 0, 0, 0, &cloud, &n, report, "kt_save_map_pcd"); if (r) return r;
    FILE* f = fopen(path, "wb");
    if (!f) { set_error("kt_save_map_pcd: cannot open %s", path); return KT_ERR_INVALID; }
    fprintf(f, "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z rgb normal_x normal_y normal_z curvature\n"
               "SIZE 4 4 4 4 4 4 4 4\nTYPE F F F F F F F F\nCOUNT 1 1 1 1 1 1 1 1\nWIDTH %zu\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\n"
               "POINTS %zu\nDATA binary\n", n, n);
    std::vector<unsigned char> buf;
    bool ok = true;
    const size_t CH = 1 << 16;
    for (size_t b = 0; b < n && ok; b += CH) {                     // x86 / aarch64 hosts are little-endian: the fields' raw bytes
        const size_t k = std::min(CH, n - b);
        buf.resize(k * 32);
        for (size_t i = 0; i < k; ++i) {
            const kt_point_xyzrgbnormal& p = cloud[b + i];
            unsigned char* o = &buf[i * 32];
            std::memcpy(o, &p.x, 12); std::memcpy(o + 12, &p.b, 4); std::memcpy(o + 16, &p.nx, 12); std::memcpy(o + 28, &p.curvature, 4);
        }
        ok = fwrite(buf.data(), 1, buf.size(), f) == buf.size();
    }
    if (fclose(f) != 0) ok = false;
    if (!ok) { set_error("kt_save_map_pcd: writing %s failed", path); return KT_ERR_CUDA; }
    return KT_OK;
}

// The map as one mesh (kt_get_map_mesh, kt_save_map_ply; the header describes which / weld).  The mesh goes to verts / tris (up to the
// capacities), or, with gv / gt, to host vectors sized to the full counts.  Device work, if any, runs on the slice stream with scratch
// that is freed before returning; nothing the tracker reads is written.
static int map_mesh(kt_ctx* c, int which, bool weld, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris,
                    std::vector<kt_mesh_vertex>* gv, std::vector<uint32_t>* gt, size_t* n_verts, size_t* n_tris, kt_weld_report* report, const char* who)
{
    kt_weld_report R; std::memset(&R, 0, sizeof(R));
    if (report) *report = R;
    *n_verts = 0; *n_tris = 0;
    if (which != 0 && which != 1) { set_error("%s: which must be 0 (recorded map) or 1 (corrected map)", who); return KT_ERR_INVALID; }
    if (c->world > 1) { set_error("%s: a volume shared by %d GPUs cannot be meshed", who, c->world); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    if (c->stream_slices) KT_CUDA(cudaStreamSynchronize(c->stream_slices));           // every slice has landed in its pinned buffers
    // slices [0, covered) come from the deformed copies; with which = 1 the later ones are moved rigidly and follow them
    const size_t covered = which == 1 ? c->deformed.size() : c->slices.size();
    std::vector<size_t> ids, voff(1, 0), toff(1, 0);
    size_t n_fixed = 0;
    for (size_t i = 0; i < c->slices.size(); ++i) {
        const SliceRec& s = c->slices[i];
        if (!s.has_mesh) continue;
        ids.push_back(i); voff.push_back(voff.back() + s.mesh_nv); toff.push_back(toff.back() + s.mesh_nt);
        if (i < covered) n_fixed += s.mesh_nv; else ++R.moved_meshes;
    }
    if (ids.empty()) { set_error("%s: no slice was recorded with meshing on (kt_set_slice_meshing)", who); return KT_ERR_STATE; }
    if (which == 1 && c->deformed.empty()) { set_error("%s: no kt_deform_map / kt_close_loop has deformed the map since the last reset", who); return KT_ERR_STATE; }
    const size_t nv = voff.back(), nt = toff.back(), rec = sizeof(kt_mesh_vertex);
    R.meshes = (int)ids.size(); R.input_verts = nv; R.input_tris = nt;
    if (nv > 0xffffffffull) { set_error("%s: %zu vertices do not fit 32-bit indices", who, nv); return KT_ERR_CAPACITY; }
    auto src = [&](size_t i) -> const kt_mesh_vertex* { return which == 1 && i < covered ? c->deformed[i].mesh_verts : c->slices[i].mesh_verts; };
    auto sized = [&](size_t ov, size_t ot) {
        R.output_verts = ov; R.output_tris = ot;
        if (gv) { gv->resize(ov); gt->resize(3 * ot); verts = gv->data(); tris = gt->data(); max_verts = ov; max_tris = ot; }
        if (!verts) max_verts = 0;
        if (!tris) max_tris = 0;
    };
    auto concat_tris = [&]() {                                       // the slices' triangles, indices offset by the vertices before them
        for (size_t k = 0; k < ids.size() && toff[k] < max_tris; ++k) {
            const SliceRec& s = c->slices[ids[k]];
            const size_t m = std::min(s.mesh_nt, max_tris - toff[k]);
            for (size_t j = 0; j < 3 * m; ++j) tris[3 * toff[k] + j] = s.mesh_tris[j] + (uint32_t)voff[k];
        }
    };
    if (!weld && n_fixed == nv) {                                    // a concatenation of pinned host buffers
        sized(nv, nt);
        for (size_t k = 0; k < ids.size() && voff[k] < max_verts; ++k)
            std::memcpy(verts + voff[k], src(ids[k]), std::min(voff[k + 1], max_verts) * rec - voff[k] * rec);
        concat_tris();
    } else {
        cudaStream_t s = c->stream_slices;
        Allocations mem(s);
        cudaEvent_t ev[4];
        for (int e = 0; e < 4; ++e) if (mem.event(&ev[e], cudaEventDefault, who)) return KT_ERR_CUDA;
        kt_mesh_vertex* d_v = 0; kt_mesh_vertex* d_ov = 0; int32_t* d_e = 0; int32_t* d_c = 0; uint32_t* d_t = 0; uint32_t* d_ot = 0;
        if (mem.device(&d_v, std::max(nv, (size_t)1), who) ||
            (weld && (mem.device(&d_e, 4 * std::max(nv, (size_t)1), who) || mem.device(&d_c, 4 * std::max(nt, (size_t)1), who) ||
                      mem.device(&d_t, 3 * std::max(nt, (size_t)1), who) || mem.device(&d_ov, std::max(nv, (size_t)1), who) ||
                      mem.device(&d_ot, 3 * std::max(nt, (size_t)1), who)))) return KT_ERR_CUDA;
        std::vector<int32_t> edges, cells;
        if (weld) {                                                  // the keys' global form, expanded on the host from the compact local keys
            edges.resize(4 * nv); cells.resize(4 * nt);
            for (size_t k = 0; k < ids.size(); ++k) {
                const SliceRec& sl = c->slices[ids[k]];
                slice_mesh_keys(sl, edges.data() + 4 * voff[k], sl.mesh_nv, cells.data() + 4 * toff[k], sl.mesh_nt);
            }
        }
        KT_CUDA(cudaEventRecord(ev[0], s));
        for (size_t k = 0; k < ids.size(); ++k) {
            const SliceRec& sl = c->slices[ids[k]];
            if (sl.mesh_nv) KT_CUDA(cudaMemcpyAsync(d_v + voff[k], src(ids[k]), sl.mesh_nv * rec, cudaMemcpyHostToDevice, s));
            if (weld && sl.mesh_nt) KT_CUDA(cudaMemcpyAsync(d_t + 3 * toff[k], sl.mesh_tris, sl.mesh_nt * 3 * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
        }
        if (weld) {
            if (nv) KT_CUDA(cudaMemcpyAsync(d_e, edges.data(), edges.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
            if (nt) KT_CUDA(cudaMemcpyAsync(d_c, cells.data(), cells.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        }
        KT_CUDA(cudaEventRecord(ev[1], s));
        if (n_fixed < nv) { int r = rigid_move_mesh(d_v + n_fixed, nv - n_fixed, map_correction(c), s); if (r) return r; }
        size_t ov = nv, ot = nt;
        if (weld) {
            kt_weld_report W;
            int r = weld_meshes(d_v, d_e, voff.data(), d_t, d_c, toff.data(), (int)ids.size(), d_ov, nv, d_ot, nt, &ov, &ot, &W, s); if (r) return r;
            R.repeated_cells = W.repeated_cells; R.dropped_triangles = W.dropped_triangles; R.merged_vertices = W.merged_vertices;
            R.sort_ms = W.sort_ms; R.weld_ms = W.weld_ms;
        }
        sized(ov, ot);
        KT_CUDA(cudaEventRecord(ev[2], s));
        const size_t kv = std::min(ov, max_verts), kt = std::min(ot, max_tris);
        if (kv) KT_CUDA(cudaMemcpyAsync(verts, weld ? d_ov : d_v, kv * rec, cudaMemcpyDeviceToHost, s));
        if (weld && kt) KT_CUDA(cudaMemcpyAsync(tris, d_ot, kt * 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        KT_CUDA(cudaEventRecord(ev[3], s));
        if (!weld) concat_tris();
        KT_CUDA(cudaStreamSynchronize(s));
        KT_CUDA(cudaEventElapsedTime(&R.upload_ms, ev[0], ev[1]));
        KT_CUDA(cudaEventElapsedTime(&R.download_ms, ev[2], ev[3]));
        KT_CUDA(cudaEventElapsedTime(&R.total_ms, ev[0], ev[3]));
    }
    *n_verts = R.output_verts; *n_tris = R.output_tris;
    if (report) *report = R;
    return KT_OK;
}

int kt_get_map_mesh(kt_ctx* c, int which, int weld, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris, size_t* n_verts,
                    size_t* n_tris, kt_weld_report* report)
{
    if (!c || !n_verts || !n_tris) { set_error("kt_get_map_mesh: bad argument"); return KT_ERR_INVALID; }
    return map_mesh(c, which, weld != 0, verts, verts ? max_verts : 0, tris, tris ? max_tris : 0, 0, 0, n_verts, n_tris, report, "kt_get_map_mesh");
}

int kt_save_map_ply(kt_ctx* c, const char* path, int which, int weld, kt_weld_report* report)
{
    if (!c || !path) { set_error("kt_save_map_ply: bad argument"); return KT_ERR_INVALID; }
    std::vector<kt_mesh_vertex> v; std::vector<uint32_t> t;
    size_t nv = 0, nt = 0;
    int r = map_mesh(c, which, weld != 0, 0, 0, 0, 0, &v, &t, &nv, &nt, report, "kt_save_map_ply"); if (r) return r;
    return write_mesh_ply(path, std::vector<PlyPart>(1, PlyPart{v.data(), nv, t.data(), nt}), "kt_save_map_ply");
}

int kt_set_map_volume(kt_ctx* c, int enabled, size_t max_bricks)
{
    const char* who = "kt_set_map_volume";
    if (!c) return KT_ERR_INVALID;
    if (c->world > 1) { set_error("%s: a volume shared by %d GPUs has no map volume", who, c->world); return KT_ERR_INVALID; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    if (!enabled) {
        if (c->mapvol) { KT_CUDA(cudaStreamSynchronize(c->stream)); c->mapvol.reset(); }
        c->mapvol_restore = false;
        return KT_OK;
    }
    std::unique_ptr<MapVolume> m(new MapVolume());
    int r = mapvol_init(m.get(), max_bricks, c->stream); if (r) return r;        // a refusal leaves the current store (or none) in place
    KT_CUDA(cudaStreamSynchronize(c->stream));
    c->mapvol = std::move(m);
    return KT_OK;
}

static int map_volume_on(kt_ctx* c, const char* who)
{
    if (c->world > 1) { set_error("%s: a volume shared by %d GPUs has no map volume", who, c->world); return KT_ERR_INVALID; }
    if (!c->mapvol) { set_error("%s: the map volume is off (kt_set_map_volume)", who); return KT_ERR_STATE; }
    KT_CUDA(cudaSetDevice(c->cfg.device));
    return KT_OK;
}

int kt_set_map_volume_restore(kt_ctx* c, int enabled)
{
    if (!c) return KT_ERR_INVALID;
    int r = map_volume_on(c, "kt_set_map_volume_restore"); if (r) return r;
    c->mapvol_restore = enabled != 0;                           // read by the next shift on the host: no device work here
    return KT_OK;
}

int kt_get_map_volume_info(kt_ctx* c, size_t* bricks, size_t* capacity, int* full)
{
    if (!c || !bricks || !capacity || !full) { set_error("kt_get_map_volume_info: bad argument"); return KT_ERR_INVALID; }
    int r = map_volume_on(c, "kt_get_map_volume_info"); if (r) return r;
    *capacity = c->mapvol->capacity;
    return mapvol_info(c->mapvol.get(), bricks, full, c->stream);
}

int kt_get_map_volume_bricks(kt_ctx* c, uint64_t* keys, int16_t* tsdf, uint8_t* color, size_t max_bricks, size_t* n_bricks)
{
    if (!c || !n_bricks) { set_error("kt_get_map_volume_bricks: bad argument"); return KT_ERR_INVALID; }
    int r = map_volume_on(c, "kt_get_map_volume_bricks"); if (r) return r;
    return mapvol_bricks(c->mapvol.get(), (unsigned long long*)keys, tsdf, color, max_bricks, n_bricks, c->stream);
}

// The map mesh into host memory: up to the capacities (verts / tris may be null), or, with gv / gt, into host vectors of the full size
static int global_mesh(kt_ctx* c, int weight_cull, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris,
                       std::vector<kt_mesh_vertex>* gv, std::vector<uint32_t>* gt, size_t* n_verts, size_t* n_tris, kt_global_mesh_report* report,
                       const char* who)
{
    kt_global_mesh_report R; std::memset(&R, 0, sizeof(R));
    if (report) *report = R;
    *n_verts = 0; *n_tris = 0;
    int r = map_volume_on(c, who); if (r) return r;
    cudaStream_t s = c->stream;
    Allocations out(s);
    kt_mesh_vertex* d_v = 0; uint32_t* d_t = 0;
    const bool fetch = gv || verts || tris;
    const MeshOutput sink = [&](size_t nv, size_t nt, void** v, uint32_t** t) -> int {
        if (!fetch) return 1;
        if (out.device(&d_v, nv, who) || out.device(&d_t, 3 * nt, who)) return KT_ERR_CUDA;
        *v = d_v; *t = d_t;
        return 0;
    };
    size_t nv = 0, nt = 0;
    float3 vs = make_float3(c->size, c->size, c->size);
    if ((r = mapvol_mesh(c->mapvol.get(), c->tsdf, c->color, c->cfg.vol, c->voxelWrap, vs, weight_cull, sink, &nv, &nt, &R, s))) return r;
    if (gv) { gv->resize(nv); gt->resize(3 * nt); verts = gv->data(); tris = gt->data(); max_verts = nv; max_tris = nt; }
    const size_t kv = verts ? std::min(nv, max_verts) : 0, kt = tris ? std::min(nt, max_tris) : 0;
    if (kv || kt) {
        cudaEvent_t ev[2];
        for (int e = 0; e < 2; ++e) if (out.event(&ev[e], cudaEventDefault, who)) return KT_ERR_CUDA;
        KT_CUDA(cudaEventRecord(ev[0], s));
        if (kv) KT_CUDA(cudaMemcpyAsync(verts, d_v, kv * sizeof(kt_mesh_vertex), cudaMemcpyDeviceToHost, s));
        if (kt) KT_CUDA(cudaMemcpyAsync(tris, d_t, kt * 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        KT_CUDA(cudaEventRecord(ev[1], s));
        KT_CUDA(cudaStreamSynchronize(s));
        KT_CUDA(cudaEventElapsedTime(&R.download_ms, ev[0], ev[1]));
        R.total_ms += R.download_ms;
    }
    *n_verts = nv; *n_tris = nt;
    if (report) *report = R;
    return KT_OK;
}

int kt_get_global_mesh(kt_ctx* c, int weight_cull, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris, size_t* n_verts,
                       size_t* n_tris, kt_global_mesh_report* report)
{
    if (!c || !n_verts || !n_tris) { set_error("kt_get_global_mesh: bad argument"); return KT_ERR_INVALID; }
    return global_mesh(c, weight_cull, verts, max_verts, tris, max_tris, 0, 0, n_verts, n_tris, report, "kt_get_global_mesh");
}

int kt_save_global_mesh_ply(kt_ctx* c, const char* path, int weight_cull, kt_global_mesh_report* report)
{
    if (!c || !path) { set_error("kt_save_global_mesh_ply: bad argument"); return KT_ERR_INVALID; }
    std::vector<kt_mesh_vertex> v; std::vector<uint32_t> t;
    size_t nv = 0, nt = 0;
    int r = global_mesh(c, weight_cull, 0, 0, 0, 0, &v, &t, &nv, &nt, report, "kt_save_global_mesh_ply"); if (r) return r;
    return write_mesh_ply(path, std::vector<PlyPart>(1, PlyPart{v.data(), nv, t.data(), nt}), "kt_save_global_mesh_ply");
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
    const void* src = which == 0 ? (void*)c->fe.maps.vmaps[level] : which == 1 ? (void*)c->fe.maps.nmaps[level] :
                      which == 2 ? (void*)c->vmaps_g_prev[level] : which == 3 ? (void*)c->nmaps_g_prev[level] :
                      which == 4 ? (void*)c->fe.maps.depths[level] : which == 5 ? (void*)c->vmap_curr_color :
                      which == 6 ? (void*)c->fe.depth_scaled : which == 7 ? (void*)c->fe.cw : (void*)c->fe.rgbf;      // 6-8: integration inputs, level 0
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
    int r = frontend_pyramid(photometric_frontend(c, depth_dev, rgb_dev, &c->ph_last), c->stream); if (r) return r;
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
    const PhotometricPyramid* ph = c->cfg.odometry != 0 ? &c->ph_next : 0;
    OdomMaps maps = {c->fe.maps.vmaps, c->fe.maps.nmaps, vmaps_g_prev4, nmaps_g_prev4};
    if (vmaps_curr4 && nmaps_curr4) {
        // the caller's current maps (createVMap / createNMap of its own pyramid); the photometric set still comes from the frame
        if (ph && (r = frontend_pyramid(photometric_frontend(c, depth_dev, rgb_dev, ph), c->stream))) return r;
        maps.vmaps_curr = vmaps_curr4; maps.nmaps_curr = nmaps_curr4;
    } else if ((r = build_frontend(c, depth_dev, rgb_dev, c->fe, 0, ph, c->stream))) return r;
    M3 Rp, Rc; V3 tp, tc;
    for (int k = 0; k < 9; ++k) Rp.m[k] = Rprev9[k];
    for (int k = 0; k < 3; ++k) tp.v[k] = tprev3[k];
    Rc = Rp; tc = tp;
    if ((r = run_odometry(c, maps, Rp, tp, &Rc, &tc))) return r;
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
    int r = c->view.grow(P * 8, P * 8, "kt_get_live_image"); if (r) return r;
    uint8_t* shaded = c->view.get(); uint8_t* col = shaded + P * 3; uint16_t* dep = (uint16_t*)(shaded + P * 6);
    const float light[3] = {c->size * -3.f, c->size * -3.f, c->size * -3.f};
    const M3 Rinv = m3_inverse(c->rmats.back());
    r = generate_views(c->vmaps_g_prev[0], c->nmaps_g_prev[0], c->vmap_curr_color, c->cfg.rows, c->cfg.cols, light, 1,
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
    const int V = c->cfg.vol;
    int lo[3] = {0, 0, 0}, hi[3] = {V, V, V};
    int r;
    if ((r = wait_slice_download(c)) || (r = fetch_cloud(c, lo, hi))) return r;
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

int kt_alloc_pinned(void** ptr, size_t bytes) { return host_malloc(ptr, bytes, "kt_alloc_pinned"); }
int kt_free_pinned(void* ptr) { if (ptr) KT_CUDA(host_free(ptr)); return KT_OK; }

} // extern "C"
