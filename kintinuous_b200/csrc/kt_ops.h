// kintinuous_b200 -- internal C++ launch API (one function per operator; the C ABI in kt_capi.cu and
// the tracker in kt_tracker.cu call these).  All pointers are device pointers, compact pitch.
#pragma once
#include "kt_common.cuh"

struct kt_deform_report;
struct kt_pgo_report;

namespace kt {

static const int LEVELS = 4;                 // ICPOdometry.h:52 / RGBDOdometry.h:96
static const int MAX_GPUS = 8;

// How the kernels reach the volume when it is shared by `world` GPUs (one process per GPU, peers mapped through CUDA IPC / NVLink).
//   * the TSDF plane (2 B / voxel) is REPLICATED: every rank holds all V^3 shorts; the owner of a voxel computes its update and stores a
//     CHANGED value into every replica (P2P stores inside integrate_kernel), so ray casting -- ~100 dependent scattered TSDF reads per
//     ray -- never leaves local HBM;
//   * the colour / weight plane (4 B / voxel, the weight in .w) is SHARDED by storage z plane, block-cyclically: planes are dealt to the
//     ranks in blocks of 2^bshift (owner = (sz >> bshift) mod world), so that whatever part of the volume the camera looks at, every
//     rank owns an equal share of the voxels to integrate; it is read remotely only for the trilinear colour tap of a ray's hit point
//     and for the neighbour voxels of an extraction at block edges.
// Ownership is a property of the STORAGE plane, hence invariant under volume shifting.  Single GPU: world = 1 (owner 0, local plane = sz).
struct VolumeView {
    int16_t* tsdf[MAX_GPUS];      // every rank's full replica (V^3 shorts); [rank] is local memory
    uint8_t* color[MAX_GPUS];     // every rank's own colour planes (V^2 * V / world uchar4), local plane order
    int world, rank, bshift, nshift;
};
__host__ __device__ __forceinline__ int vv_owner(const VolumeView& v, int sz) { return (sz >> v.bshift) & (v.world - 1); }
__host__ __device__ __forceinline__ int vv_local_plane(const VolumeView& v, int sz)
{ return ((sz >> (v.bshift + v.nshift)) << v.bshift) | (sz & ((1 << v.bshift) - 1)); }
inline VolumeView single_volume(int16_t* tsdf, uint8_t* color, int V)
{
    (void)V;
    VolumeView v; for (int g = 0; g < MAX_GPUS; ++g) { v.tsdf[g] = tsdf; v.color[g] = color; }
    v.world = 1; v.rank = 0; v.bshift = 0; v.nshift = 0;
    return v;
}

// ---- pyramid (kt_pyramid.cu) ----
int bilateral(const uint16_t* src, uint16_t* dst, int rows, int cols, cudaStream_t s);
int pyrdown(const uint16_t* src, uint16_t* dst, int src_rows, int src_cols, cudaStream_t s);
int create_vmap(const Intr& k, const uint16_t* depth, float* vmap, int rows, int cols, cudaStream_t s);
int create_nmap(const float* vmap, float* nmap, int rows, int cols, cudaStream_t s);
struct MapsLevel { const uint16_t* depth; float* vmap; float* nmap; int rows, cols; Intr k; float fx_inv, fy_inv;
                   const float* vstale; const float* nstale; };   // maps of the previous frame when the output is a spare set (Q7), else null
int create_maps_pyramid(const MapsLevel* levels, int n_levels, cudaStream_t s);      // fused vmap+nmap, all levels, one launch
int transform_maps(const float* vs, const float* ns, const Mat33& R, const float3& t, float* vd, float* nd, int rows, int cols, cudaStream_t s);
struct TransformLevel { const float* vs; const float* ns; float* vd; float* nd; int rows, cols; };
int transform_maps_pyramid(const TransformLevel* levels, int n_levels, const Mat33& R, const float3& t, cudaStream_t s);
int resize_map(const float* in, float* out, int in_rows, int in_cols, bool normalize, cudaStream_t s);

// ---- fused front end (kt_frontend.cu): depth pyramid, vertex / normal maps of all levels, colour prep, photometric pyramids + gradients ----
struct FrontendArgs {
    const uint16_t* depth_f;       // bilateral-filtered depth, level 0 (null: no depth pyramid / maps, photometric set only)
    const uint16_t* depth_raw;     // raw depth (photometric set)
    const uint8_t* rgb;            // colour prep + intensity
    int rows, cols; Intr k;
    uint16_t* const* depths;       // [LEVELS]; [0] is depth_f itself (not written)
    float* const* vmaps; float* const* nmaps; float* const* vstale; float* const* nstale;      // [LEVELS] each; stale may be null
    float* cw; float4* rgbf; bool angle_color;                                                   // colour prep outputs (null: skip)
    int cut_off; float* const* depth_m; uint8_t* const* intensity; int16_t* const* dIdx; int16_t* const* dIdy;   // photometric set (null: skip)
};
int frontend_pyramid(const FrontendArgs& a, cudaStream_t s);
// bilateralFilter + scaleDepth in one launch (they share the raw-depth tile); either output may be null
int bilateral_scale(const uint16_t* src, uint16_t* dst, float* scaled, int rows, int cols, const Intr& k, bool angle_color, cudaStream_t s);

// ---- GUI taps (kt_views.cu): generateImage + generateDepth in one launch; any of the three outputs may be null ----
int generate_views(const float* vmap, const float* nmap, const uint8_t* vmap_color, int rows, int cols, const float* light_pos3, int n_lights,
                   uint8_t* dst_rgb, uint8_t* dst_color_rgb, const float* Rinv9, const float* t3, uint16_t* depth, cudaStream_t s);

// ---- RGB-D preprocessing (kt_rgb.cu) ----
int short_depth_to_metres(const uint16_t* src, float* dst, int rows, int cols, int cut_off, cudaStream_t s);
int pyrdown_gauss_f(const float* src, float* dst, int src_rows, int src_cols, cudaStream_t s);
int bgr_to_intensity(const uint8_t* rgb, uint8_t* dst, int rows, int cols, cudaStream_t s);
int pyrdown_uchar_gauss(const uint8_t* src, uint8_t* dst, int src_rows, int src_cols, cudaStream_t s);
int derivative_images(const uint8_t* src, int16_t* dx, int16_t* dy, int rows, int cols, cudaStream_t s);
int project_to_point_cloud(const float* depth, float* cloud, int rows, int cols, double fx, double fy, double cx, double cy, cudaStream_t s);

// ---- odometry reductions (kt_icp.cu, kt_rgb.cu) ----
// Device-resident Gauss-Newton state shared by all iterations of one frame.
struct OdomState {
    // inputs of the frame
    float Rprev[9], tprev[3], Rprev_inv[9];
    // running estimate (ICPOdometry.cpp:73-74,177-178)
    float Rcurr[9], tcurr[3];
    int odo_timeout;                        // set by a whole-frame kernel whose exchange poll gave up (a peer CTA never arrived); read back with the pose
    double resultRt[16];                    // cv::Mat resultRt (ICPOdometry.cpp:83)
    // photometric warp of the current iteration (RGBDOdometry.cpp:209-231)
    float krkinv[9], kt[3];
    int rgb_count, rgb_sigma;               // computeRgbResidual outputs
    float sums_icp[32], sums_rgb[32];       // reduced [JtJ|Jtr] (27) + residual + inliers
    int iter;                               // iterations done this frame
    unsigned int blocks_done;               // last-block-done counter
    unsigned int blocks_done_rgb;
};
static const int TRACE_STRIDE = 44;          // A(36) b(6) residual(2)
static const int MAX_PARTIALS = 1024;

struct IcpLevelArgs {
    const float* vmap_curr; const float* nmap_curr; const float* vmap_g_prev; const float* nmap_g_prev;
    int rows, cols; Intr k; float dist_thres, angle_thres;
};
// One ICP normal-equation build + (optionally) the on-device solve and pose update.
//   mode 0: reduce only, result left in state->sums_icp (used by the operator API and by -ri before rgb_step)
//   mode 1: reduce + LDLT solve + pose update on device (ICP-only odometry)
int icp_iteration(const IcpLevelArgs& a, OdomState* state, float* partials, float* trace, int mode, cudaStream_t s);

// peer_words / world / rank (optional): the exchange words of every rank of a shared volume (NVLink peer memory) -- the pixel rows of every
// level are then split over the ranks and the 29 sums are all-reduced inside the kernel (grid_sum_words_mg, kt_frame.cuh)
int icp_frame(const IcpLevelArgs* levels, const int* iters, const float* pose12_host, OdomState* state, unsigned long long* xwords_dev,
              float* trace, int* timeout_dev, long long* prof_dev, float* host_pose, unsigned int host_seq, cudaStream_t s,
              unsigned long long* const* peer_words = 0, int world = 1, int rank = 0);
// exchange words of the whole-frame odometry kernels (grid_sum_words, kt_frame.cuh): their count, and the reset (zero) of a word array --
// stream-ordered, once per frame between two odometry launches
size_t odom_exchange_words();          // allocation size (64-bit words)
int odom_exchange_used(int* stride);   // number of words actually used, and their spacing
int odom_exchange_reset(unsigned long long* xwords_dev, cudaStream_t s);

struct RgbLevelArgs {
    const int16_t* dIdx; const int16_t* dIdy; const float* last_depth; const float* next_depth;
    const uint8_t* last_image; const uint8_t* next_image; void* corres; const float* cloud;
    int rows, cols; float min_scale, max_depth_delta, fx, fy, sobel_scale; double Kfx, Kfy, Kcx, Kcy;
};
// use_state_warp 1: (K R K^-1, K t) rebuilt on the device from state->resultRt; 0: taken from state->krkinv / kt
int rgb_residual(const RgbLevelArgs& a, OdomState* state, int* partials, int use_state_warp, cudaStream_t s);
// mode 0: reduce only; 1: solve RGB-only; 2: solve A_rgb + 100 A_icp (RGBDOdometry.cpp:316-321)
// Returns 1 (and launches nothing) when the image does not fit the kernel's shared-memory stage.  xwords_dev: zero at launch (see icp_frame).
int rgbd_frame(const IcpLevelArgs* icp_levels, const RgbLevelArgs* rgb_levels, const int* iters, int with_icp, const float* pose12_host, OdomState* state,
               unsigned long long* xwords_dev, float* trace, int* timeout_dev, float* host_pose, unsigned int host_seq, cudaStream_t s);
int rgb_iteration(const RgbLevelArgs& a, OdomState* state, float* partials, float* trace, int mode, float sigma_override, cudaStream_t s);
// pose12_dev: Rprev (9) + tprev (3) in device memory
int odom_begin_frame(OdomState* state, const float* pose12_dev, cudaStream_t s);
int reduce_grid_for(int n_items);

// ---- volume (kt_tsdf.cu, kt_raycast.cu, kt_extract.cu) ----
int init_volume(int16_t* tsdf, uint8_t* color, int vol, cudaStream_t s);                  // whole volume
int init_shared(const VolumeView& vv, int vol, cudaStream_t s);       // this rank's TSDF replica and colour planes
int clear_volume(int axis, int back, int16_t* tsdf, uint8_t* color, int vol, int current_wrap, int delta_wrap, cudaStream_t s);
// shared volume: the TSDF planes of the local replica and the colour planes this rank owns
int clear_volume_shared(int axis, int back, const VolumeView& vv, int vol, int current_wrap, int delta_wrap, cudaStream_t s);
int scale_depth(const uint16_t* depth, float* scaled, int rows, int cols, const Intr& k, bool angle_color, cudaStream_t s);
struct IntegrateArgs {
    const float* depth_scaled; int rows, cols; Intr k; float3 volume_size; Mat33 Rinv; float3 t; float trunc;
    int16_t* tsdf; uint8_t* color; int vol; int3 wrap; const uint8_t* rgb; const float* nmap_curr; bool angle_color;
    int multi; VolumeView vv;    // multi != 0: the volume is shared by vv.world GPUs (tsdf / color above are vv.tsdf[rank] / vv.color[rank])
    float* cw; float4* rgbf;     // optional per-pixel scratch (rows*cols each): colour weight + float RGB prepared once per frame
    unsigned long long* reset_words; int reset_count, reset_stride;   // optional: reset_count 64-bit words, reset_stride apart, that the launch zeroes (the odometry's exchange words)
};
int integrate(const IntegrateArgs& a, float* ztable_dev /* 2*vol floats */, cudaStream_t s);
// per-pixel colour weight (sign = normal invalid) + float RGB for IntegrateArgs::cw / rgbf; once per frame, after the normal map exists
int color_prep(const float* nmap, const uint8_t* rgb, int rows, int cols, bool angle_color, float* cw, float4* rgbf, cudaStream_t s);
struct RaycastArgs {
    Intr k; Mat33 R; float3 t; float trunc; float3 volume_size; const int16_t* tsdf; const uint8_t* color; int vol; int3 wrap;
    float* vmap[LEVELS]; float* nmap[LEVELS]; int rows, cols; uint8_t* vmap_color; int n_levels;   // n_levels>1: fused model pyramid
    // multi-GPU (world > 1): rays read any slab through vv, this rank casts the tile rows [tile_row_begin, tile_row_end) and stores
    // its results into EVERY rank's model maps (P2P stores = the all-gather, fused into the kernel epilogue)
    int multi; VolumeView vv; int tile_row_begin, tile_row_end;
    float* peer_vmap[MAX_GPUS][LEVELS]; float* peer_nmap[MAX_GPUS][LEVELS]; uint8_t* peer_vcol[MAX_GPUS];
};
int raycast(const RaycastArgs& a, cudaStream_t s);
int extract_slice(const int16_t* tsdf, const float3& volume_size, int vol, void* out, size_t capacity, const int3& wrap,
                  const uint8_t* color, int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int subsample,
                  const int3& real_wrap, unsigned int* counter_dev, cudaStream_t s);
// shared volume: only voxels whose storage plane this rank owns emit points; colours of foreign planes are read through vv (P2P)
int extract_slice_mg(const VolumeView& vv, const float3& volume_size, int vol, void* out, size_t capacity, const int3& wrap,
                     int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int subsample,
                     const int3& real_wrap, unsigned int* counter_dev, cudaStream_t s);
// ---- slice post-processing (kt_slice.cu): CloudSliceProcessor.cpp:97-162 on the device ----
struct SliceWorkspace { unsigned int* mask; unsigned int* word_off; unsigned int* block_tot; size_t words_cap; void* acc; size_t acc_cap; unsigned int* bounds; unsigned int* bounds_host; };
int process_slice(const void* points_dev /* kt_point_xyzrgb */, size_t n, int weight_cull, float leaf, int k_search, void* out_dev /* kt_point_xyzrgbnormal */,
                  size_t capacity, size_t* count, SliceWorkspace* ws, cudaStream_t s);
void slice_ws_free(SliceWorkspace* ws);
// ---- marching cubes over a box of the cyclic volume (kt_mesh.cu): an indexed mesh in a fixed order, see the file header ----
struct MeshArgs {
    const int16_t* tsdf; const uint8_t* color; int vol; float3 volume_size; int3 wrap; int3 real_wrap;   // wrap / real_wrap: as extract_slice
    int minX, maxX, minY, maxY, minZ, maxZ; int weight_cull;
};
struct MeshWorkspace {
    unsigned long long* counts; size_t counts_cap;    // per-tile vertex / triangle totals and their exclusive scans
    void* tmp; size_t tmp_cap;                        // CUB scan storage
    unsigned long long* keys; size_t keys_cap;        // 3 * owner + axis of every vertex, ascending
    unsigned long long* totals_host;                  // pinned: vertex and triangle counts
    MeshWorkspace() : counts(0), counts_cap(0), tmp(0), tmp_cap(0), keys(0), keys_cap(0), totals_host(0) {}
};
// count + scan, then one read-back (synchronises s): the mesh's vertex and triangle counts
int mesh_count(const MeshArgs& a, MeshWorkspace* ws, size_t* n_verts, size_t* n_tris, cudaStream_t s);
// after mesh_count with the same arguments: writes n_verts 32-byte kt_mesh_vertex records and the triangles (3 x uint32 each); asynchronous
int mesh_emit(const MeshArgs& a, MeshWorkspace* ws, size_t n_verts, void* verts, uint32_t* tris, cudaStream_t s);
void mesh_ws_free(MeshWorkspace* ws);
// ---- embedded deformation graph (kt_deform.cu, host logic in kt_deform.hpp) ----
// Node positions: float n x 3 (device), node times ascending.  kind: 0 kt_point_xyzrgbnormal, 1 kt_mesh_vertex, 2 packed float xyz.
// Writes 4 node ids (int32, ascending) and 4 FP64 weights per point; asynchronous.
int deform_weights(const float* node_pos, const uint64_t* node_times, int n_nodes, const void* pts, int kind, const uint64_t* times, size_t n,
                   int32_t* ids, double* weights, cudaStream_t s);
// Gauss-Newton over the graph (host arrays: node positions, constraint sources / targets and their ids / weights); writes the 12
// unknowns per node (rotation column-major, translation) to x_dev -- the identity unless rep->deformed -- and every field of the
// report.  Synchronises s.
int deform_optimise(const float* node_pos, int n_nodes, const float* src, const double* dst, const int32_t* ids, const double* weights, size_t m,
                    double* x_dev, kt_deform_report* rep, cudaStream_t s);
// Deforms n records of kind 0 / 1 from in to out (may not alias) with the nodes' unknowns x; asynchronous.
int deform_apply(const float* node_pos, const double* x, int n_nodes, const int32_t* ids, const double* weights, const void* in, void* out,
                 int kind, size_t n, cudaStream_t s);
// ---- pose-graph optimisation (kt_pgo.cu, host logic in kt_pgo.hpp) ----
struct PgoFactor;
// Gauss-Newton from poses_in (device, n x 16 FP64) into X (device, may alias) over the host factor list; every field of the report.
// Synchronises s.
int pgo_optimise(const double* poses_in, int n, const PgoFactor* factors, int n_factors, double* X, kt_pgo_report* rep, cudaStream_t s);
// cross-GPU barrier: every rank writes `epoch` into slot [rank] of every peer's flag array, then waits until all slots of its own
// array reach `epoch` (bounded spin: returns through *error_dev != 0 instead of hanging the GPU if a peer never arrives)
int xgpu_barrier(unsigned int* const* peer_flags_dev /* [world] device array of pointers */, unsigned int* my_flags, int rank, int world,
                 unsigned int epoch, int* error_dev, cudaStream_t s);

} // namespace kt
