// kintinuous_b200 -- internal C++ launch API (one function per operator; the C ABI in kt_capi.cu and
// the tracker in kt_tracker.cu call these).  All pointers are device pointers, compact pitch.
#pragma once
#include "kt_common.cuh"
#include "kt_mem.hpp"
#include <functional>

struct kt_deform_report;
struct kt_pgo_report;
struct kt_weld_report;
struct kt_global_mesh_report;

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
// shared volume: zero the storage planes [first, first + planes) (mod vol) along `axis` that clear_range gives, in the local TSDF
// replica and the colour planes this rank owns
int clear_volume_shared(int axis, const VolumeView& vv, int vol, int first, int planes, cudaStream_t s);
// the storage planes [first, first + planes) (mod vol) along `axis` that clear_volume zeroes (SURVEY.md Q13: an x clear reaches round_up_16)
void clear_range(int axis, int back, int vol, int current_wrap, int delta_wrap, int* first, int* planes);
int scale_depth(const uint16_t* depth, float* scaled, int rows, int cols, const Intr& k, bool angle_color, cudaStream_t s);
struct IntegrateArgs {
    const float* depth_scaled; int rows, cols; Intr k; float3 volume_size; Mat33 Rinv; float3 t; float trunc;
    int16_t* tsdf; uint8_t* color; int vol; int3 wrap; const uint8_t* rgb; const float* nmap_curr; bool angle_color;
    int multi; VolumeView vv;    // multi != 0: the volume is shared by vv.world GPUs (tsdf / color above are vv.tsdf[rank] / vv.color[rank])
    float* cw; float4* rgbf;     // optional per-pixel scratch (rows*cols each): colour weight + float RGB prepared once per frame
    unsigned long long* reset_words; int reset_count, reset_stride;   // optional: reset_count 64-bit words, reset_stride apart, that the launch zeroes (the odometry's exchange words)
};
int integrate(const IntegrateArgs& a, float* ztable_dev /* 2*vol floats */, cudaStream_t s);
struct RaycastArgs {
    Intr k; Mat33 R; float3 t; float trunc; float3 volume_size; const int16_t* tsdf; const uint8_t* color; int vol; int3 wrap;
    float* vmap[LEVELS]; float* nmap[LEVELS]; int rows, cols; uint8_t* vmap_color; int n_levels;   // n_levels>1: fused model pyramid
    // multi-GPU (world > 1): rays read any slab through vv, this rank casts the tile rows [tile_row_begin, tile_row_end) and stores
    // its results into EVERY rank's model maps (P2P stores = the all-gather, fused into the kernel epilogue)
    int multi; VolumeView vv; int tile_row_begin, tile_row_end;
    float* peer_vmap[MAX_GPUS][LEVELS]; float* peer_nmap[MAX_GPUS][LEVELS]; uint8_t* peer_vcol[MAX_GPUS];
};
int raycast(const RaycastArgs& a, cudaStream_t s);
int check_cell_size(const float3& volume_size, int vol);      // raycast()'s refusal of a cell size it cannot divide by (-1, error set)
int extract_slice(const int16_t* tsdf, const float3& volume_size, int vol, void* out, size_t capacity, const int3& wrap,
                  const uint8_t* color, int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int subsample,
                  const int3& real_wrap, unsigned int* counter_dev, cudaStream_t s);
// shared volume: only voxels whose storage plane this rank owns emit points; colours of foreign planes are read through vv (P2P)
int extract_slice_mg(const VolumeView& vv, const float3& volume_size, int vol, void* out, size_t capacity, const int3& wrap,
                     int minX, int maxX, int minY, int maxY, int minZ, int maxZ, int subsample,
                     const int3& real_wrap, unsigned int* counter_dev, cudaStream_t s);
// ---- slice post-processing (kt_slice.cu): CloudSliceProcessor.cpp:97-162 on the device ----
struct SliceWorkspace {
    DeviceBuffer<unsigned int> mask, word_off, block_tot;    // leaf bitmap, its word offsets and scan block totals (grown together)
    DeviceBuffer<unsigned char> acc;                         // per-leaf accumulators
    Allocations fixed; unsigned int* bounds = nullptr; unsigned int* bounds_host = nullptr;
};
int process_slice(const void* points_dev /* kt_point_xyzrgb */, size_t n, int weight_cull, float leaf, int k_search, void* out_dev /* kt_point_xyzrgbnormal */,
                  size_t capacity, size_t* count, SliceWorkspace* ws, cudaStream_t s);
// ---- marching cubes over a box of the cyclic volume (kt_mesh.cu): an indexed mesh in a fixed order, see the file header ----
struct MeshArgs {
    const int16_t* tsdf; const uint8_t* color; int vol; float3 volume_size; int3 wrap; int3 real_wrap;   // wrap / real_wrap: as extract_slice
    int minX, maxX, minY, maxY, minZ, maxZ; int weight_cull;
};
struct MeshWorkspace {
    DeviceBuffer<unsigned long long> counts;          // per-tile vertex / triangle totals and their exclusive scans
    DeviceBuffer<unsigned char> tmp;                  // CUB scan storage
    DeviceBuffer<unsigned long long> keys;            // 3 * owner + axis of every vertex, ascending
    Allocations fixed; unsigned long long* totals_host = nullptr;      // pinned: vertex and triangle counts
};
// count + scan, then one read-back (synchronises s): the mesh's vertex and triangle counts
int mesh_count(const MeshArgs& a, MeshWorkspace* ws, size_t* n_verts, size_t* n_tris, cudaStream_t s);
// after mesh_count with the same arguments: writes n_verts 32-byte kt_mesh_vertex records and the triangles (3 x uint32 each); asynchronous.
// vkeys (may be null: the workspace's): receives every vertex's local key 3 * owner + axis; tcells (may be null): every triangle's cell
// as the owner-grid index of its lower corner.  Neither changes the vertices or triangles.
int mesh_emit(const MeshArgs& a, MeshWorkspace* ws, size_t n_verts, void* verts, uint32_t* tris, cudaStream_t s, unsigned long long* vkeys = nullptr,
              unsigned long long* tcells = nullptr);
// What turns a box's local keys into global voxels: the owner grid's origin and x / y extents, and the box's real_wrap.
struct MeshKeyFrame { int min[3]; int ex, ey; int real_wrap[3]; };
MeshKeyFrame mesh_key_frame(const MeshArgs& a);
// owner-grid index -> (gx, gy, gz, axis): the logical voxel plus real_wrap, the world voxel index the positions are computed from
__host__ __device__ inline void mesh_key_global(const MeshKeyFrame& f, unsigned long long owner, int axis, int32_t* g)
{
    const unsigned long long r = owner / (unsigned long long)f.ex;
    g[0] = f.min[0] + (int)(owner % (unsigned long long)f.ex) + f.real_wrap[0];
    g[1] = f.min[1] + (int)(r % (unsigned long long)f.ey) + f.real_wrap[1];
    g[2] = f.min[2] + (int)(r / (unsigned long long)f.ey) + f.real_wrap[2];
    g[3] = axis;
}
// n local keys -> n int32 x 4 global ones (edges: vertex keys, else triangle cells); asynchronous
int mesh_global_keys(const MeshArgs& a, const unsigned long long* keys, size_t n, bool edges, int32_t* out, cudaStream_t s);
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
// ---- place recognition (kt_surf.cu, kt_place.cu, cloud_fitness in kt_slice.cu; host logic in kt_place.hpp) ----
struct SurfWorkspace {          // sized for one image shape
    int rows = 0, cols = 0; Allocations mem;
    int* integral = nullptr; float* resp = nullptr; void* cand = nullptr; unsigned long long* keys = nullptr; unsigned int* idx = nullptr;
    unsigned int* n_cand = nullptr; unsigned char* tmp = nullptr; size_t tmp_bytes = 0;
};
int surf_ws_reserve(SurfWorkspace* ws, int rows, int cols);
// RGB image -> at most max_features keypoints, strongest first: kp 6 floats each (x, y, size, angle in radians, response, laplacian sign),
// desc 64 floats each, *n_out_dev (device) = keypoints written.  Asynchronous.
int surf(const uint8_t* rgb, int rows, int cols, float threshold, int max_features, float* kp, float* desc, int* n_out_dev, SurfWorkspace* ws, cudaStream_t s);
// camera-frame xyz of each keypoint (kt_place.hpp place_lookup_3d), NaN without one; max_n rows written
int keypoints_3d(const float* kp, const int* n_dev, int max_n, const uint16_t* depth, int rows, int cols, const Intr& k, float* xyz, cudaStream_t s);
// n_seg segments of `stride` database rows (64 floats each), segment g's first seg_count_dev[g] valid; per row the two nearest of the first
// *n_query_dev (<= q_cap) query descriptors: best index, d1, d2 (squared), pass = d1 < ratio d2; seg_passes (may be null): passes per segment
int match_ratio(const float* db, int n_seg, int stride, const int* seg_count_dev, const float* q, const int* n_query_dev, int q_cap, float ratio,
                int* best, float* d1, float* d2, unsigned char* pass, int* seg_passes, cudaStream_t s);
struct PnpArgs { const float* p_new; const float* p_old; const float* uv_old; int n; Intr k; int iterations; float threshold_px; unsigned long long seed; };
struct PnpWorkspace { DeviceBuffer<int> counts; DeviceBuffer<double> hyps; DeviceBuffer<unsigned int> counter; };
// pose12 (device, FP64): R row-major + t with R p_new + t in the old camera; inliers (device) per match; *n_inliers (device)
int pnp_ransac(const PnpArgs& a, PnpWorkspace* ws, double* pose12, unsigned char* inliers, int* n_inliers, cudaStream_t s);
// depth (u16 mm) -> rows*cols kt_point_xyzrgb, alpha 1 where the depth is valid
int depth_to_cloud(const uint16_t* depth, int rows, int cols, const Intr& k, void* cloud, cudaStream_t s);
// getFitnessScore of the loop check: d2_dev holds capacity + 8 doubles; synchronises s
int cloud_fitness(const void* src, size_t n_src, const void* dst, size_t n_dst, float leaf, const float* T12, SliceWorkspace* ws_src, SliceWorkspace* ws_dst,
                  void* src_out, void* dst_out, size_t capacity, double* d2_dev, double* fitness, size_t* n_src_used, size_t* n_dst_used, cudaStream_t s);
// ---- whole-map export (kt_map.cu) ----
// pcl::VoxelGrid (downsample_all_data) over n records of kind 0 (kt_point_xyzrgb) or 1 (kt_point_xyzrgbnormal): one centroid per leaf in
// ascending 64-bit leaf index, the first min(leaves, capacity) written to out (may be null), *count = leaves; *pcl_would_skip = PCL's
// int64 overflow check fired (PCL would return the input unfiltered).  ms2 (may be null): device ms of keys + sort, of leaf starts +
// centroids.  Workspace allocated and freed per call; synchronises s.
int voxel_grid(const void* points_dev, size_t n, int kind, float leaf, void* out_dev, size_t capacity, size_t* count, int* pcl_would_skip,
               float* ms2, cudaStream_t s);
struct RigidF { float R[9]; float t[3]; };       // row-major rotation and translation
// x' = R x + t and n' = R n of n kt_point_xyzrgbnormal records in place, FP32 without contraction; asynchronous
int rigid_move(void* points_dev, size_t n, const RigidF& C, cudaStream_t s);
// the same move of n kt_mesh_vertex records in place
int rigid_move_mesh(void* verts_dev, size_t n, const RigidF& C, cudaStream_t s);
// ---- mesh weld (kt_weld.cu): n_meshes keyed meshes concatenated -> one mesh, every global cell and edge once; see the file header ----
// voff / toff: n_meshes + 1 host offsets into the vertices / triangles.  rep: every field but upload_ms / download_ms.  Scratch
// allocated and freed per call; synchronises s.
int weld_meshes(const void* verts, const int32_t* vert_edges, const size_t* voff, const uint32_t* tris, const int32_t* tri_cells, const size_t* toff,
                int n_meshes, void* out_verts, size_t max_verts, uint32_t* out_tris, size_t max_tris, size_t* n_verts, size_t* n_tris,
                kt_weld_report* rep, cudaStream_t s);
// ---- map volume (kt_mapvol.cu): a sparse global TSDF of the voxels the shifts clear, 8^3 bricks behind a hash; see the file header ----
static const int MAPVOL_BRICK_VOXELS = 512;      // voxel (x, y, z) of a brick at x + 8 y + 64 z
static const int MAPVOL_COORD_BIAS = 1 << 20;    // brick key: (bz + bias) << 42 | (by + bias) << 21 | (bx + bias), 21 bits per axis
struct MapVolume {
    Allocations mem;
    unsigned int capacity = 0, slots = 0;                                    // bricks; hash slots (a power of two >= 2 capacity)
    unsigned long long* slot_key = nullptr; unsigned int* slot_val = nullptr;  // open addressing, empty = ~0; value = pool index
    unsigned long long* brick_key = nullptr;                                 // pool index -> key
    int16_t* tsdf = nullptr; uint8_t* color = nullptr;                       // pool: 512 voxels per brick
    unsigned int* state = nullptr; unsigned int* state_host = nullptr;       // bricks taken, committed, refused, full
};
// allocates everything up front (KT_ERR_CUDA when refused) and empties it
int mapvol_init(MapVolume* m, size_t max_bricks, cudaStream_t s);
int mapvol_empty(MapVolume* m, cudaStream_t s);
// before a clear of storage planes [first, first + planes) along axis (clear_range): keep their voxels; wrap = the signed voxel wrap.
// Three launches, asynchronous.
int mapvol_store(MapVolume* m, const int16_t* tsdf, const uint8_t* color, int vol, const int* wrap, int axis, int first, int planes, cudaStream_t s);
// after that clear: every voxel of the same planes whose global voxel under wrap_after (the signed wrap once this axis has moved) has a
// stored value with W != 0 takes it; the others stay cleared.  One launch, asynchronous; the volume is written, never read.
int mapvol_restore(MapVolume* m, int16_t* tsdf, uint8_t* color, int vol, const int* wrap_after, int axis, int first, int planes, cudaStream_t s);
int mapvol_info(MapVolume* m, size_t* bricks, int* full, cudaStream_t s);          // synchronises s
// the store sorted by key into host arrays (any may be null); *n = bricks; KT_ERR_CAPACITY beyond max.  Synchronises s.
int mapvol_bricks(MapVolume* m, unsigned long long* keys, int16_t* tsdf, uint8_t* color, size_t max, size_t* n, cudaStream_t s);
// Where a mesh goes once its counts are known: return 0 with device pointers for nv vertices and nt triangles, 1 for the counts alone,
// or a negative kt_status.
using MeshOutput = std::function<int(size_t nv, size_t nt, void** verts, uint32_t** tris)>;
struct BrickSet { const unsigned long long* keys; const int16_t* tsdf; const uint8_t* color; size_t n; };   // device, keys strictly ascending
// marching cubes over a brick set (kt_mesh.cu's contract with the global voxel as the logical one, no border; positions with real wrap
// 0 and centred by vol); ms (may be null): device ms of count + emit, of the sorts, in all.  Scratch per call; synchronises s.
int mesh_bricks(const BrickSet& set, const float3& volume_size, int vol, int weight_cull, const MeshOutput& out, size_t* n_verts, size_t* n_tris,
                float* ms, cudaStream_t s);
// the map mesh: mesh_bricks over the store merged with the live volume (wrap = the signed voxel wrap); every field of the report but
// download_ms.  Synchronises s.
int mapvol_mesh(const MapVolume* m, const int16_t* tsdf, const uint8_t* color, int vol, const int* wrap, const float3& volume_size, int weight_cull,
                const MeshOutput& out, size_t* n_verts, size_t* n_tris, kt_global_mesh_report* rep, cudaStream_t s);
// cross-GPU barrier: every rank writes `epoch` into slot [rank] of every peer's flag array, then waits until all slots of its own
// array reach `epoch` (bounded spin: returns through *error_dev != 0 instead of hanging the GPU if a peer never arrives)
int xgpu_barrier(unsigned int* const* peer_flags_dev /* [world] device array of pointers */, unsigned int* my_flags, int rank, int world,
                 unsigned int epoch, int* error_dev, cudaStream_t s);

} // namespace kt
