/*
 * kintinuous_b200 -- C ABI of the H100-native dense tracking-and-fusion hot path.
 *
 * This header is the drop-in boundary (SURVEY.md section 8b): plain pointers and sizes, no torch /
 * Eigen / OpenCV / PCL types.  Each entry point names the reference interface it replaces
 * (paths relative to mp3guy/Kintinuous, src/frontend/).  The source-compatible C++ shim that
 * re-creates the reference class / free-function names on top of this ABI is
 * include/kintinuous_b200_shim.hpp; INTEGRATION.md shows how a maintainer wires it in.
 *
 * Conventions
 *   - every function returns KT_OK (0) or a negative kt_status; kt_last_error() gives the text.
 *     The reference's cudaSafeCall prints and exit(0)s (cuda/internal.h:76-86); this ABI never exits.
 *   - "dev" pointers are device pointers on the context's GPU, images are compact row-major
 *     (pitch = cols * sizeof(T)); vertex / normal maps are the reference's SoA layout: three float
 *     planes x,y,z stacked vertically, 3*rows x cols (KintinuousTracker.cpp:373-377).
 *   - Mat33 arguments are 9 floats row-major (Eigen::Matrix<float,3,3,RowMajor>, device_cast<Mat33>,
 *     cuda/internal.h:481-485); float3 arguments are 3 floats; Intr is {fx, fy, cx, cy}.
 *   - stream arguments are cudaStream_t passed as void* (NULL = the context's / default stream).
 *   - there is NO CPU fallback: without a CUDA device every call fails with KT_ERR_CUDA.
 */
#ifndef KINTINUOUS_B200_H_
#define KINTINUOUS_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define KT_API __attribute__((visibility("default")))
#else
#define KT_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef enum kt_status {
    KT_OK = 0,
    KT_ERR_INVALID = -1,   /* bad argument / unsupported configuration */
    KT_ERR_CUDA = -2,      /* CUDA runtime error (text in kt_last_error) */
    KT_ERR_STATE = -3,     /* call out of order */
    KT_ERR_CAPACITY = -4   /* output buffer too small */
} kt_status;

/* Replaces: the ConfigArgs flags the path reads (utils/ConfigArgs.h:111-185), Volume / Resolution
 * singletons (Volume.h:26-57, Resolution.h:23-69), the cv::Mat K of KintinuousTracker(cv::Mat*)
 * (KintinuousTracker.cpp:71-91) and the compile-time VOL macro (cuda/internal.h:243). */
typedef struct kt_config {
    int rows, cols;          /* Resolution (480 x 640) */
    float fx, fy, cx, cy;    /* depth intrinsics (MainController.cpp:222-227) */
    int vol;                 /* voxels per side; runtime here, '#define VOL 512' in the reference */
    float volume_size;       /* metres, -s (default 6) */
    int odometry;            /* 0 = ICP (default), 1 = RGB-D (-r), 2 = ICP + RGB-D (-ri) */
    int fast_odometry;       /* -fod */
    int voxel_shift;         /* -t (default 14) */
    int overlap;             /* setOverlap (TrackerInterface.h:58, default 2) */
    int angle_color;         /* !disableColorAngleWeight (-dc) */
    int parked;              /* setParked / static mode: never shift */
    int cloud_capacity;      /* slice point buffer; 0 = 3*rows*cols (KintinuousTracker.cpp:77) */
    int device;              /* CUDA device ordinal (-gpu) */
    /* multi-GPU z-slab sharding (no counterpart in the reference; SURVEY.md section 8e) */
    int rank, world;         /* this process' rank / number of ranks sharing ONE volume (1 = single GPU) */
} kt_config;

typedef struct kt_pose {
    float R[9];              /* camera -> volume rotation, row-major (rmats_.back()) */
    float t[3];              /* camera position in the volume frame, metres (tvecs_.back()) */
    float global_t[3];       /* currentGlobalCamera (KintinuousTracker.cpp:581-596) */
    int voxel_wrap[3];       /* signed accumulated wrap (voxelWrap) */
    int shifted;             /* number of CloudSlices produced by this frame */
    int frame;               /* global_time_ after the frame */
} kt_pose;

/* 32-byte point, byte-compatible with pcl::PointXYZRGB / cuda/internal.h:156-184 */
typedef struct kt_point_xyzrgb {
    float x, y, z, _pad0;
    uint8_t b, g, r, a;
    uint8_t _pad1[12];
} kt_point_xyzrgb;

/* 48-byte point, byte-compatible with pcl::PointXYZRGBNormal: what CloudSliceProcessor hands to the deformation / meshing backend
 * (backend/CloudSliceProcessor.cpp:162, CloudSlice::processedCloud, CloudSlice.h:57). */
typedef struct kt_point_xyzrgbnormal {
    float x, y, z, data3;            /* data3 = 1 (PCL's homogeneous coordinate) */
    float nx, ny, nz, data_n3;
    uint8_t b, g, r, a;
    float curvature;
    float pad[2];
} kt_point_xyzrgbnormal;

/* 32-byte mesh vertex (kt_op_mesh_volume, kt_get_slice_mesh): position in the slice frame (metres, as kt_point_xyzrgb), unit normal
 * towards increasing TSDF (free space; (0,0,0) when degenerate), colour and alpha = weight of the voxel nearer the surface. */
typedef struct kt_mesh_vertex {
    float x, y, z, nx, ny, nz;
    uint8_t r, g, b, a;
    uint32_t _pad;
} kt_mesh_vertex;

typedef struct kt_ctx kt_ctx;

KT_API const char* kt_last_error(void);
/* 1 when the library was built with the sm_90a kernels and a CUDA device is usable. */
KT_API int kt_cuda_available(void);

/* ---- tracker: replaces class KintinuousTracker (KintinuousTracker.h:85-172) ---- */
KT_API int kt_create(const kt_config* cfg, kt_ctx** out);                 /* KintinuousTracker::KintinuousTracker (.cpp:71-182) */
KT_API int kt_destroy(kt_ctx* ctx);                                       /* ~KintinuousTracker (.cpp:184-197) */
KT_API int kt_reset(kt_ctx* ctx);                                         /* KintinuousTracker::reset (.cpp:262-354) */
/* KintinuousTracker::processFrame (.cpp:444-915) together with the upload its caller does
 * (backend/TrackerInterface.cpp:90-91).  depth: rows*cols u16 mm; rgb: rows*cols*3 u8 (PixelRGB r,g,b).
 * Host buffers (pinned memory from kt_alloc_pinned makes the copy asynchronous). */
KT_API int kt_process_frame(kt_ctx* ctx, const uint16_t* depth_host, const uint8_t* rgb_host, uint64_t utime, kt_pose* out);
/* Optional hint: start on the NEXT frame now.  Its copy into spare input buffers and its pose-independent front end (scaleDepth,
 * bilateral filter, depth pyramid, vertex / normal maps) run on a side stream and overlap the fusion / ray-cast of the current frame.
 * A following kt_process_frame / kt_process_frame_device with the same two pointers consumes the prefetched set; with other pointers
 * the hint is dropped.  Host (pinned, for an asynchronous copy) or device pointers; the buffers must stay valid and unchanged until
 * that call.  Results are bit-identical with or without the hint. */
KT_API int kt_prefetch_frame(kt_ctx* ctx, const uint16_t* depth, const uint8_t* rgb);
/* Same, inputs already resident in device memory (DeviceArray2D arguments of processFrame). */
KT_API int kt_process_frame_device(kt_ctx* ctx, const uint16_t* depth_dev, const uint8_t* rgb_dev, uint64_t utime, kt_pose* out);
KT_API int kt_finalise(kt_ctx* ctx);                                      /* KintinuousTracker::finalise (.cpp:1003-1048) */
KT_API int kt_get_pose(kt_ctx* ctx, kt_pose* out);                        /* getLastRotation/getLastTranslation/getVolumeOffset */
KT_API float kt_get_voxel_size(kt_ctx* ctx);                              /* getVoxelSize */
KT_API float kt_get_trunc_dist(kt_ctx* ctx);                              /* TsdfVolume::getTsdfTruncDist (TSDFVolume.cpp:125-129) */
KT_API int kt_set_overlap(kt_ctx* ctx, int overlap);                      /* setOverlap */
KT_API int kt_set_parked(kt_ctx* ctx, int parked);                        /* setParked */
/* getCloudSlices (.cpp:1055-1058): slices stay owned by the context until kt_reset / kt_destroy. */
KT_API int kt_num_slices(kt_ctx* ctx);
/* Copies up to max_points points of slice idx; *count = the slice's size; dimension = CloudSlice::Dimension
 * (CloudSlice.h:33-44: XPlus..ZMinus, FIRST, FINAL, TSDF); camera_t = 3 floats, may be NULL. */
KT_API int kt_get_slice(kt_ctx* ctx, int idx, kt_point_xyzrgb* points, size_t max_points, size_t* count, int* dimension, float* camera_t);
/* CloudSliceProcessor on the device (backend/CloudSliceProcessor.cpp:97-162; kt_op_process_slice below): when enabled, every slice
 * recorded from now on is also culled by weight (alpha >= weight_cull, the reference's -cw, default 8), voxel-grid filtered at one
 * voxel and given 20-nearest-neighbour normals BEFORE it leaves the GPU; kt_get_processed_slice returns CloudSlice::processedCloud.
 * Slices are downloaded asynchronously into pinned memory; both getters wait for the slice they are asked for, not for the tracker. */
KT_API int kt_set_slice_processing(kt_ctx* ctx, int enabled, int weight_cull);
KT_API int kt_get_processed_slice(kt_ctx* ctx, int idx, kt_point_xyzrgbnormal* points, size_t max_points, size_t* count);
/* The rest of the CloudSlice record (CloudSlice.h:47-60): which odometry produced the pose (CloudSlice::Odometry: 0 ICP, 2 RGBD --
 * KintinuousTracker.cpp:137-176,565: the kind of the active OdometryProvider), the camera pose at hand-over (volume-global
 * translation, row-major rotation) and the frame's timestamp. */
/* Meshing on the device, standing in for MeshGenerator (backend/MeshGenerator.cpp:37-191 the meshing thread, :193-227 calculateMesh,
 * :229-280 save).  The reference triangulates every slice's processed cloud with PCL's greedy projection on the CPU; here each slice is
 * meshed by marching cubes over the TSDF box it was extracted from, before that box is cleared (kt_op_mesh_volume below: no parity with
 * PCL).  When enabled, every slice recorded from now on carries a mesh (weight_cull: corners need alpha >= weight_cull, -cw, default
 * 8); the FINAL slice of kt_finalise meshes the whole volume.  Neighbouring slices overlap by the overlap planes, so their meshes
 * repeat the triangles there (as the reference's merged export with default flags keeps its overlap).  kt_get_slice_mesh copies up to
 * max_verts / max_tris and returns both counts; it waits for that slice's download only, and returns KT_ERR_STATE for a slice recorded
 * with meshing off.  A volume shared by several GPUs (world > 1) cannot be meshed: KT_ERR_INVALID. */
KT_API int kt_set_slice_meshing(kt_ctx* ctx, int enabled, int weight_cull);
KT_API int kt_get_slice_mesh(kt_ctx* ctx, int idx, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris,
                             size_t* n_verts, size_t* n_tris);
/* The whole volume's mesh at this moment, synchronous, without recording a slice (the live mesh of PangoVis.cpp:395), with the weight
 * cull of kt_set_slice_meshing (8 until it is called); copies up to the capacities, returns both counts.  world > 1: KT_ERR_INVALID. */
KT_API int kt_get_live_mesh(kt_ctx* ctx, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris, size_t* n_verts, size_t* n_tris);
/* Where slice idx's mesh sits on the global voxel lattice (the keys kt_get_map_mesh welds by): per vertex (gx, gy, gz, axis), the lower
 * voxel and axis of the edge it lies on; per triangle (gx, gy, gz, 0), the lower corner of its cell -- the logical voxel plus the slice's
 * real voxel wrap, the world voxel index the positions are computed from (kt_op_mesh_volume_keyed).  Copies up to max_verts / max_tris
 * records of 4 int32 (the counts are kt_get_slice_mesh's); waits for that slice's download only.  KT_ERR_STATE for a slice recorded
 * with meshing off. */
KT_API int kt_get_slice_mesh_keys(kt_ctx* ctx, int idx, int32_t* vert_edges, size_t max_verts, int32_t* tri_cells, size_t max_tris);
/* MeshGenerator::save's "merging for export" branch (:229-280): every recorded slice mesh in order, indices offset, as one binary
 * little-endian PLY (vertex: float x y z nx ny nz, uchar red green blue; face: list uchar int vertex_indices).  KT_ERR_STATE when no
 * recorded slice has a mesh. */
KT_API int kt_save_mesh_ply(kt_ctx* ctx, const char* path);
typedef struct kt_slice_info { int dimension; int odometry; float camera_t[3]; float camera_R[9]; uint64_t utime; size_t count; } kt_slice_info;
KT_API int kt_get_slice_info(kt_ctx* ctx, int idx, kt_slice_info* info);
/* Dense pose graph (KintinuousTracker::DensePose / densePoseGraph / latestDensePoseId, KintinuousTracker.h:151-172): one record per
 * processed frame -- the frame's timestamp, the 4x4 camera pose [R | currentGlobalCamera] (row-major) and the loop-pose flag (true for the
 * first frame, KintinuousTracker.cpp:534) -- what the deformation backend samples (backend/Deformation.cpp:134-169). */
typedef struct kt_dense_pose { uint64_t timestamp; float pose[16]; int is_loop_pose; } kt_dense_pose;
KT_API int kt_num_dense_poses(kt_ctx* ctx);                                /* latestDensePoseId */
KT_API int kt_get_dense_pose(kt_ctx* ctx, int idx, kt_dense_pose* out);    /* densePoseGraph.at(idx) */
/* Map deformation to a corrected trajectory: the embedded deformation graph of the reference's backend (backend/Deformation.cpp:173-346
 * addCameraLoop, backend/DeformationGraph.cpp) on the GPU.  Loop detection and the pose-graph solve (iSAM) stay with the caller: it passes
 * the corrected camera poses, each with a timestamp that is in the dense pose graph (else KT_ERR_INVALID), and optional point constraints
 * (its loop-closure inliers: time, position in the map as tracked, where it belongs).
 *   - Nodes: the dense pose graph's camera positions, the first and then every one more than node_spacing from the last taken
 *     (initialiseGraphPoses, DeformationGraph.cpp:51-86; the reference's -dg, default 0.8 m), joined sequentially (connectGraphSeq).
 *     Fewer than 5 nodes: KT_ERR_STATE.
 *   - Constraints: each corrected pose pulls the tracked camera position at its time to the corrected one (positions only, as the
 *     reference); each point constraint pulls its source to its target.
 *   - Gauss-Newton (optimiseGraphSparse, :714-774): at most 10 steps; no step at all when |r_con| / constraints < 0.1.
 *   - The map is every processed slice (kt_set_slice_processing) and every slice mesh (kt_set_slice_meshing) recorded so far; a vertex's
 *     time is its slice's.  The deformed copies are kept in new pinned memory (kt_get_deformed_slice / _mesh); the recorded slices are not
 *     modified.  Every call deforms the original map from scratch with the constraints it is given -- the reference deforms its map in
 *     place, loop closure after loop closure.
 * KT_ERR_STATE with neither processed slices nor meshes; KT_ERR_INVALID for a volume shared by several GPUs (world > 1) and for a
 * corrected translation, point source or point target that is not finite. */
typedef struct kt_deform_constraint { uint64_t time; float source[3]; float target[3]; } kt_deform_constraint;
typedef struct kt_deform_report {
    int nodes, constraints;
    int band;                   /* widest node-id span of a term, in 12 x 12 blocks of J^T J (at most 19) */
    int iterations;             /* Gauss-Newton steps taken */
    double initial_error;       /* |r|^2 before the first step */
    double final_error;         /* |r|^2 after the last one */
    double constraint_error;    /* |r_con| / constraints before the first step (the early-out test: < 0.1) */
    int deformed;               /* 0: the map is returned unchanged (early-out or failed factorisation) */
    int solver_failed;          /* 1: a pivot of the Cholesky factorisation was not positive */
} kt_deform_report;
KT_API int kt_deform_map(kt_ctx* ctx, const kt_dense_pose* corrected, size_t n, const kt_deform_constraint* points, size_t n_points,
                         float node_spacing, kt_deform_report* report);
/* The deformed processed cloud / mesh vertices of slice idx as of the last kt_deform_map (the triangles are kt_get_slice_mesh's).  Copy
 * up to the capacity, return the count.  KT_ERR_STATE for a slice recorded after that call or without a processed cloud / mesh. */
KT_API int kt_get_deformed_slice(kt_ctx* ctx, int idx, kt_point_xyzrgbnormal* points, size_t max_points, size_t* count);
KT_API int kt_get_deformed_slice_mesh(kt_ctx* ctx, int idx, kt_mesh_vertex* verts, size_t max_verts, size_t* n_verts);
/* The "_opt" mesh of Deformation::saveMesh (Deformation.cpp:85-100): kt_save_mesh_ply's layout over the deformed vertices of the slices
 * covered by the last kt_deform_map.  KT_ERR_STATE before any kt_deform_map or when none of those slices has a mesh. */
KT_API int kt_save_deformed_mesh_ply(kt_ctx* ctx, const char* path);
/* The map as one point cloud: the files a run exists to produce (MainController.cpp:238-265).
 *   which = 0, the recorded map (CloudSliceProcessor::save, CloudSliceProcessor.cpp:180-231): the processed cloud of every slice recorded
 *     with slice processing on since the last reset, in order, the FINAL slice of kt_finalise included.
 *   which = 1, the corrected map (Deformation::saveCloud, Deformation.cpp:67-83): the slices covered by the last kt_deform_map /
 *     kt_close_loop contribute their deformed copies (kt_get_deformed_slice); every slice recorded after it is moved rigidly by that
 *     deformation's last correction C = P_corr(t) P_tracked(t)^-1, with t the last corrected pose passed to kt_deform_map (the identity
 *     when it was given point constraints only) or the last pose-graph node of kt_close_loop -- what iSAM's odometry chain gives a pose
 *     after the last loop (Deformation::addVertices, :421-457).  Positions x' = R x + t and normals n' = R n in FP32 on the device (the
 *     reference's pcl::transformPointCloud leaves the normals unrotated).  KT_ERR_STATE before any deformation or after kt_reset.
 *   dedupe = 1 is the reference's -nos: pcl::VoxelGrid at kt_get_voxel_size over the whole concatenation (kt_op_voxel_grid), which merges
 *     the points that neighbouring slices repeat in their overlap planes.  Without it the recorded map is copied on the host, no GPU work.
 * kt_get_map_cloud copies up to `capacity` points (out may be NULL: the count alone) and returns the full count; every call redoes the
 * work, so a count-then-fetch pair costs two exports.  It waits for slice downloads still in flight and works on the slice stream
 * between frames: tracking reads nothing it writes.  kt_save_map_pcd writes the same cloud as PCL 1.7.2's savePCDFile(path, cloud, true):
 * the ASCII header (FIELDS x y z rgb normal_x normal_y normal_z curvature, DATA binary), then 32 packed little-endian bytes per point in
 * field order (rgb = the b, g, r, a bytes).  The reference's files: "<log>.pcd" = (which 0, dedupe -nos), "<log>_opt.pcd" = (which 1,
 * dedupe 0).  KT_ERR_STATE when no slice was recorded with slice processing on; KT_ERR_INVALID for a volume shared by several GPUs
 * (world > 1: each rank's slices hold only its own voxels); KT_ERR_CUDA when device memory for the export cannot be allocated (nothing
 * else changes). */
typedef struct kt_map_report {
    size_t input_points;        /* points of the concatenation */
    size_t output_points;       /* points of the exported cloud (the voxel grid's leaves with dedupe) */
    int slices;                 /* slices recorded with slice processing on */
    int moved_slices;           /* slices placed by the rigid correction (which = 1) */
    int pcl_would_skip;         /* dedupe: PCL's int64 check fired, so PCL would have returned the cloud unfiltered (this export filters) */
    float upload_ms, sort_ms, centroid_ms, download_ms, total_ms;   /* CUDA-event times of the device work (0 without any) */
} kt_map_report;
KT_API int kt_get_map_cloud(kt_ctx* ctx, int which, int dedupe, kt_point_xyzrgbnormal* out, size_t capacity, size_t* count, kt_map_report* report);
KT_API int kt_save_map_pcd(kt_ctx* ctx, const char* path, int which, int dedupe, kt_map_report* report);
/* The map as one mesh, the mesh half of the export above (the reference's MeshGenerator::save, MeshGenerator.cpp:37-191).
 *   which = 0: every slice mesh recorded with meshing on since the last reset, in order, the FINAL slice of kt_finalise included.
 *   which = 1: the corrected map, as kt_get_map_cloud's: slices covered by the last kt_deform_map / kt_close_loop contribute their
 *     deformed vertices (kt_get_deformed_slice_mesh); later slices are moved rigidly by the same C (positions R x + t, normals R n, FP32
 *     on the device).  The triangles are which 0's.  KT_ERR_STATE before any deformation or after kt_reset.
 *   weld = 0: the concatenation with offset indices (kt_save_mesh_ply's content).
 *   weld = 1: kt_op_weld_meshes over the slice meshes and their keys (kt_get_slice_mesh_keys): every global cell keeps the triangles
 *     of the latest slice that meshed it (its TSDF has fused the most frames), every global edge one vertex, so the overlap planes
 *     neighbouring slices share appear once and the seams are connected.  Where two slices disagree about the sign of a shared corner
 *     (the surface moved between them) a gap one cell wide is left; there is no hole filling.
 * Copies up to max_verts / max_tris (NULL outputs: counts only) and returns both counts; every call redoes the work.  Waits for slice
 * downloads still in flight and works on the slice stream between frames: tracking reads nothing it writes.  KT_ERR_STATE when no slice
 * was recorded with meshing on; KT_ERR_INVALID for a volume shared by several GPUs; KT_ERR_CUDA when device memory for the export cannot
 * be allocated.  kt_save_map_ply writes the same mesh in kt_save_mesh_ply's binary PLY layout; the reference's "-nos" mesh is
 * (which 0, weld 1). */
typedef struct kt_weld_report {
    size_t input_verts, input_tris;     /* of the concatenation */
    size_t output_verts, output_tris;   /* of the exported mesh */
    size_t repeated_cells;              /* weld: cells that more than one mesh has triangles in */
    size_t dropped_triangles;           /* weld: triangles in a cell another, later mesh also meshed */
    size_t merged_vertices;             /* weld: vertices kept triangles use that share their edge with a later mesh's vertex */
    int meshes;                         /* slices (meshes) in the concatenation */
    int moved_meshes;                   /* slices placed by the rigid correction (which = 1) */
    float upload_ms, sort_ms, weld_ms, download_ms, total_ms;      /* CUDA-event times of the device work (0 without any) */
} kt_weld_report;
KT_API int kt_get_map_mesh(kt_ctx* ctx, int which, int weld, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris,
                           size_t* n_verts, size_t* n_tris, kt_weld_report* report);
KT_API int kt_save_map_ply(kt_ctx* ctx, const char* path, int which, int weld, kt_weld_report* report);
/* The map volume (no counterpart in the reference, which meshes point slices with PCL's GP3): a sparse global TSDF kept on the device,
 * so that the whole map is meshed in ONE marching-cubes pass over one consistent field and no seam is left open where the surface moved
 * between two slices (the weld above cannot close those: the values that would decide them were cleared at the shift).
 *   - Just before each shift clears its storage planes, the surface voxels of those planes (W != 0 and F != 1) get their 8^3 brick, and
 *     every cleared voxel with W != 0 overwrites its value in a brick that exists: each global voxel keeps its latest observation, and
 *     free space observed later removes an old surface.  A global voxel is the logical voxel plus the real voxel wrap (the index of
 *     kt_get_slice_mesh_keys).  Bricks are keyed (bz + 2^20) << 42 | (by + 2^20) << 21 | (bx + 2^20) (21 signed bits per axis, z most
 *     significant); voxel (x, y, z) of brick b is global voxel 8 b + (x, y, z), stored at x + 8 y + 64 z.
 *   - Capacity is all or nothing per cleared slab: when a slab's new bricks do not all fit, none is stored (bricks already stored are
 *     still updated), `full` is set and tracking carries on.  Three kernel launches per cleared slab on the tracker stream (four with
 *     restore, below), no host synchronisation; frames without a shift launch nothing more.  Off by default.
 * kt_set_map_volume(ctx, 1, max_bricks) allocates an empty store of max_bricks bricks (3 KB each plus 24 B of hash per brick) up front,
 * replacing any current one; KT_ERR_CUDA when the memory is refused, and then nothing else changes.  enabled = 0 frees it.  kt_reset
 * empties it.  KT_ERR_INVALID for a volume shared by several GPUs (world > 1); the calls below return KT_ERR_STATE while it is off. */
KT_API int kt_set_map_volume(kt_ctx* ctx, int enabled, size_t max_bricks);
/* Restore: the store flows back into the moving volume, so that a camera returning to mapped space tracks against the surface it fused
 * there and keeps averaging into it (instead of a blank volume, whose few new frames would later overwrite the stored surface).
 *   - A shift clears storage planes [first, first + planes) along an axis (the store's set: Q13's round_up16 reach on x and Q12's ZMinus
 *     slab included).  Once the clear has run, with wrap' the signed voxel wrap after this axis moves, every voxel of those planes whose
 *     global voxel (logical voxel + wrap') lies in a stored brick with W != 0 there takes the stored tsdf and colour words, bit for bit;
 *     every other voxel stays cleared.  Per axis, in x, y, z order: store -> clear -> restore, one more launch, no host synchronisation.
 *     A later axis of the same frame stores the voxels this one restored, which changes nothing; kt_get_global_mesh's field is unchanged.
 *   - The planes a clear reaches beyond those that leave the volume keep their global voxels, so their surface bricks come back in the
 *     same frame: with restore on, the volume (and so tracking) can differ from restore off, and from the reference, at the first shift
 *     that clears surface, even without a revisit.  Only bricks holding a surface are stored, so free space outside them is not
 *     restored: a ray through it sees cleared voxels, as after any clear.
 * Off by default; it belongs to the context and applies to the clears that follow (never to planes that entered before).  kt_reset and a
 * replacing kt_set_map_volume(ctx, 1, n) keep it, kt_set_map_volume(ctx, 0, ...) turns it off.  It is a host flag read at the next
 * shift, so it may change between any two frames.  KT_ERR_STATE while the map volume is off, KT_ERR_INVALID for world > 1. */
KT_API int kt_set_map_volume_restore(kt_ctx* ctx, int enabled);
KT_API int kt_get_map_volume_info(kt_ctx* ctx, size_t* bricks, size_t* capacity, int* full);
/* The stored bricks sorted by key: keys, tsdf (512 int16 per brick) and colour (512 x 4 uint8: b, g, r, weight per voxel, the volume's
 * layout); any output may be NULL.  *n_bricks = the count; KT_ERR_CAPACITY (nothing copied) when it exceeds max_bricks. */
KT_API int kt_get_map_volume_bricks(kt_ctx* ctx, uint64_t* keys, int16_t* tsdf, uint8_t* color, size_t max_bricks, size_t* n_bricks);
/* The whole map's mesh: kt_op_mesh_bricks over S, the store where the live volume has W = 0 and the live volume elsewhere (the live
 * volume is read, nothing is modified, so an export mid-run changes nothing that follows).  Corners need alpha >= weight_cull.  Vertices
 * ascend by (owning global voxel in (z, y, x) order, edge axis), triangles by cell in that order, then in table order: a run that never
 * shifted gives kt_get_live_mesh's bytes.  The store is in tracked coordinates (there is no corrected variant).  Copies up to max_verts /
 * max_tris (NULL outputs: counts only) and returns both counts; synchronous, on the tracker stream, scratch freed before returning.
 * kt_save_global_mesh_ply writes the same mesh in kt_save_mesh_ply's binary PLY layout. */
typedef struct kt_global_mesh_report {
    size_t bricks;                      /* bricks meshed: the store's and the live volume's surface bricks, each once */
    size_t store_bricks, live_bricks;
    size_t input_voxels;                /* bricks x 512 */
    size_t output_verts, output_tris;
    int store_full;                     /* a shift's bricks did not fit the store (kt_get_map_volume_info's full) */
    float gather_ms, mesh_ms, sort_ms, download_ms, total_ms;   /* CUDA-event times: merge of store and live volume; count + emit; sorts */
} kt_global_mesh_report;
KT_API int kt_get_global_mesh(kt_ctx* ctx, int weight_cull, kt_mesh_vertex* verts, size_t max_verts, uint32_t* tris, size_t max_tris,
                              size_t* n_verts, size_t* n_tris, kt_global_mesh_report* report);
KT_API int kt_save_global_mesh_ply(kt_ctx* ctx, const char* path, int weight_cull, kt_global_mesh_report* report);
/* Loop closure: the pose-graph half of the reference's backend (backend/Deformation.cpp:130-346 addCameraCamera / addCameraLoop,
 * backend/iSAMInterface.cpp) on the GPU.  The caller passes what PlaceRecognition produces (LoopClosureConstraint,
 * PlaceRecognition.cpp:198-209): time1 (the new frame) and time2 (the old one), both dense pose timestamps, the pose of the camera at
 * time2 in the frame of the camera at time1 (row-major 4 x 4, ~ P(time1)^-1 P(time2)) and the PnP inliers seen from each camera
 * (camera-frame xyz, n_inliers of each).  Loop detection itself stays with the caller.
 *   - Nodes: every dense pose (pose_spacing 0), or the first, each more than pose_spacing from the last taken (the reference's -fl with
 *     -dg), and every pose a loop names; the last dense pose always.  Odometry factors join consecutive nodes; one factor per loop; a
 *     prior anchors the first node at its tracked pose; covariance 1e-3 I everywhere (iSAMInterface.cpp:44-105).
 *   - Every call re-optimises the whole graph from the tracked trajectory with every accepted loop plus the new one (FP64 Gauss-Newton,
 *     at most 100 steps, until chi2 falls by less than 1e-3 or 1e-5 relative).  chi2 < isam_thresh (the reference's -it, 10) accepts
 *     the loop; otherwise nothing observable changes (Deformation.cpp:254-343).
 *   - On acceptance the map recorded so far (as kt_deform_map, node_spacing its -dg) is deformed from the original slices: each node's
 *     tracked position to its optimised one, and each inlier of every accepted loop from its tracked to its optimised position.
 *     Without processed slices or meshes only the trajectory is corrected (map_deformed = 0).
 * Every check comes first and a failed one changes nothing: times in the dense pose graph (KT_ERR_INVALID), time1 != time2, finite input,
 * a rotation within 1e-3 of orthonormal, enough deformation nodes for a recorded map (KT_ERR_STATE), at most 64 accepted loops
 * (KT_ERR_CAPACITY).  A CUDA error while the map is deformed drops the deformed copies (as kt_deform_map) and does not record the loop.
 * Tracking never reads the corrected poses.  A volume shared by several GPUs: KT_ERR_INVALID. */
typedef struct kt_loop_constraint {
    uint64_t time1, time2;
    double constraint[16];
    const float* inliers1;          /* n_inliers xyz triples in the camera at time1 (inliers1Proj); may be NULL when n_inliers == 0 */
    const float* inliers2;          /* n_inliers xyz triples in the camera at time2 (inliers2Proj) */
    size_t n_inliers;
} kt_loop_constraint;
typedef struct kt_loop_report {
    int nodes, factors, loops, iterations;
    double chi2_initial, chi2_final;    /* sum of squared whitened errors before / after the optimisation */
    int accepted;                       /* chi2_final < isam_thresh and the factorisation succeeded */
    int solver_failed;                  /* a pivot was not positive: the loop is rejected */
    int map_deformed;                   /* the deformation moved the map (deform.deformed); deform holds that run's report, which is
                                           all zero when no map is recorded or the loop is rejected */
    kt_deform_report deform;
} kt_loop_report;
KT_API int kt_close_loop(kt_ctx* ctx, const kt_loop_constraint* loop, float pose_spacing, float node_spacing, double isam_thresh,
                         kt_loop_report* report);
KT_API int kt_num_loops(kt_ctx* ctx);                                      /* accepted loops since the last reset */
/* Loop DETECTION: the reference's place-recognition thread (backend/PlaceRecognition.cpp) as two calls.
 *   - kt_set_loop_detection(ctx, p) with p->enabled = 1: from the next frame on, keyframes are captured -- the first frame, every frame
 *     whose (|rodrigues(Rcurr^-1 R_last)| + |g_curr - g_last|) / 2 >= 0.15 since the last keyframe, and every frame that shifts the volume
 *     (KintinuousTracker.cpp:605-624, 706-718).  A keyframe's raw depth is copied and its SURF keypoints / descriptors (hessian 400,
 *     4 octaves, 2 layers, 64-d) computed on a side stream, with no host synchronisation on the frame path; its dense pose gets
 *     is_loop_pose = 1.  A full store (max_keyframes) stops adding; kt_num_keyframes reports it.  Disabled (the default): nothing is
 *     allocated or launched.  NULL or enabled = 0 disables and frees the store.  Enabling allocates the store on the device up front:
 *     max_keyframes x (rows x cols x 2 B of depth + max_features x 292 B of keypoints, descriptors and 3-D points) plus a few frames of
 *     scratch -- about 0.9 GB at 640 x 480 with the defaults.
 *   - kt_detect_loops processes every keyframe captured since the last call, in order (PlaceRecognition::process): exhaustive
 *     ratio-test retrieval (0.49 on squared distances) against every keyframe at least exclude_recent older -> the one with the most
 *     passes (>= 40, ties to the older); 3-D matches of that pair (>= 40); PnP RANSAC (500 hypotheses, 2 px) with inlier ratio >
 *     inlier_ratio; the product's projective point-to-plane ICP between the two keyframes' depth maps, bootstrapped by PnP; fitness (mean
 *     squared nearest-neighbour distance of the old keyframe's 2.5-voxel-filtered cloud, aligned, to the new one's) < 0.01 m^2.  With
 *     close = 1 each loop found goes to kt_close_loop (pose_spacing, node_spacing, isam_thresh), and a loop it ACCEPTS starts the
 *     loop_throttle_s throttle (frame timestamps; keyframes within it are not tried), as the reference's backend does; a rejected loop
 *     starts none.  With close = 0 the library cannot know the outcome: every loop found starts the throttle.  One kt_place_result per keyframe, at most `capacity` (the rest stay pending); the
 *     inlier pointers of a result's constraint stay valid until the next call.  world > 1: KT_ERR_INVALID. */
typedef struct kt_loop_detection_params {
    int enabled;
    float inlier_ratio;          /* -il, 0.35 */
    double loop_throttle_s;      /* -lt, 30 (frame timestamps) */
    double isam_thresh;          /* -it, 10 */
    float node_spacing;          /* -dg, 0.8 */
    float pose_spacing;          /* -fl: 0 = every pose */
    int max_keyframes;           /* 1000 */
    int max_features;            /* 1000 per keyframe */
    int exclude_recent;          /* 20 */
    int close;                   /* 1: kt_close_loop every loop found */
} kt_loop_detection_params;
typedef enum kt_place_stage {
    KT_PLACE_LOOP = 0,           /* a loop constraint was produced */
    KT_PLACE_THROTTLED = 1,      /* within loop_throttle_s of the last loop */
    KT_PLACE_NO_CANDIDATE = 2,   /* no keyframe old enough with >= 40 ratio-test passes */
    KT_PLACE_MATCHES = 3,        /* fewer than 40 3-D matches */
    KT_PLACE_INLIERS = 4,        /* PnP inlier ratio <= inlier_ratio */
    KT_PLACE_FITNESS = 5         /* ICP fitness >= 0.01 */
} kt_place_stage;
typedef struct kt_place_result {
    int keyframe; uint64_t time;         /* the keyframe processed */
    int candidate; uint64_t candidate_time;   /* -1 / 0: none */
    int passes, matches, inliers;
    float inlier_ratio;
    double fitness;                      /* -1 when not reached */
    int stage;                           /* kt_place_stage */
    kt_loop_constraint constraint;       /* stages KT_PLACE_FITNESS and KT_PLACE_LOOP: constraint[] = the pose the fitness was measured at; KT_PLACE_LOOP: time1 = time, time2 = candidate_time, inliers */
    int closed;                          /* close = 1 and kt_close_loop accepted it */
    kt_loop_report report;               /* kt_close_loop's report (close = 1) */
} kt_place_result;
KT_API int kt_default_loop_detection(kt_loop_detection_params* p);
KT_API int kt_set_loop_detection(kt_ctx* ctx, const kt_loop_detection_params* p);
KT_API int kt_detect_loops(kt_ctx* ctx, kt_place_result* out, size_t capacity, size_t* n_out);
/* Keyframes captured since the last reset (full = 1 once the store refused one); kt_get_keyframe waits for that keyframe's capture. */
KT_API int kt_num_keyframes(kt_ctx* ctx, int* full);
KT_API int kt_get_keyframe(kt_ctx* ctx, int idx, uint64_t* timestamp, int* dense_pose_index, int* n_features);
/* The optimised nodes of the last accepted loop (timestamp, world-frame pose, is_loop_pose = named by a loop): the corrected
 * trajectory (iSAMInterface::getCameraPoses, :169-182).  0 nodes before any accepted loop. */
KT_API int kt_num_pose_graph_nodes(kt_ctx* ctx);
KT_API int kt_get_pose_graph_node(kt_ctx* ctx, int idx, kt_dense_pose* out);
/* KintinuousTracker::outputPose (.cpp:199-218, :911-914): append one line per tracked frame to `path` ("<saveFile>.poses" in the
 * reference: "utime/1e6 gx gy gz qx qy qz qw").  NULL closes the log.  kt_format_pose_line formats one such line into buf. */
KT_API int kt_set_pose_log(kt_ctx* ctx, const char* path);
KT_API int kt_format_pose_line(uint64_t timestamp, const float* global_t3, const float* R9, char* buf, size_t capacity);
/* Per-iteration normal equations of the last frame, n x 44 floats (A 6x6 row-major, b 6, residual, inliers):
 * what icpStep / rgbStep hand back to the host each iteration (cuda/reduce.cu:404-418). */
KT_API int kt_get_trace(kt_ctx* ctx, float* dst, int max_iters, int* n_iters);
/* TsdfVolume::data() / ColorVolume::data() in the reference layout: short[V^3], uchar4[V^3], x fastest,
 * storage (cyclic) order.  Either pointer may be NULL.  (TSDFVolume.h:154, ColorVolume.h:93) */
KT_API int kt_volume_export_reference_layout(kt_ctx* ctx, int16_t* tsdf_host, uint8_t* color_host);
/* which: 0 vmap_curr, 1 nmap_curr, 2 vmap_g_prev, 3 nmap_g_prev (3*rows_l*cols_l floats), 4 depth_curr (u16),
 * 5 raycast colour (uchar4, level 0); 6 scaled depth (float), 7 colour weight (float), 8 float RGB (float4): the integration's per-pixel
 * inputs, level 0.  Test / GUI tap (getLiveImage inputs). */
KT_API int kt_download_map(kt_ctx* ctx, int which, int level, void* dst_host);
/* Stage timers (CUDA events) of the last frame, milliseconds: pyramid, odometry, shift, integrate, raycast, total. */
KT_API int kt_get_stage_ms(kt_ctx* ctx, float* ms6);
KT_API int kt_set_stage_timing(kt_ctx* ctx, int enabled);
/* CUDA-event duration of the last whole-frame ICP launch (icp_frame_kernel), ms; 0 unless stage timing is on and odometry == 0 */
KT_API float kt_get_icp_kernel_ms(kt_ctx* ctx);
/* The launches alone, ms: whole-frame ICP kernel, z table + integrate, ray cast -- without the cross-GPU barriers that the stage timers
 * of a shared-volume context include (0 unless stage timing is on). */
KT_API int kt_get_kernel_ms(kt_ctx* ctx, float* ms3);
/* Device-side stopwatch on the tracker's own stream: mark(0) ... frames ... mark(1), then the CUDA-event time between the two
 * marks (ms, synchronises on mark 1; < 0 on error).  bench.py times its region with this, not with the host clock. */
KT_API int kt_span_mark(kt_ctx* ctx, int which);
KT_API float kt_span_elapsed_ms(kt_ctx* ctx);
/* ---- ONE volume shared by `world` GPUs, one process per GPU (no counterpart in the reference; SURVEY.md 8e) ----
 * The TSDF plane is replicated on every GPU (the owner of a voxel stores its changed value into all replicas over NVLink, inside the
 * integration kernel), the colour / weight plane is sharded by storage z plane, block-cyclically.  Every rank creates its context with
 * kt_config.rank / world, exports the CUDA-IPC handle (64 bytes) of its shared arena (TSDF replica, colour planes, model maps, barrier
 * flags), the host exchanges the handles (torch.distributed / MPI / anything) and every rank calls kt_mgpu_connect with all `world`
 * handles in rank order.  After that kt_process_frame must be called by all ranks with the same frame; results (poses, model maps,
 * TSDF replicas) are bit-identical on every rank and to the single-GPU run.  With world > 1, kt_volume_export_reference_layout and
 * the slices cover the storage planes this rank owns (kt_mgpu_info: info5 = world, rank, planes owned, planes per ownership block,
 * arena MB; local plane l is storage plane (l / B * world + rank) * B + l % B). */
KT_API int kt_mgpu_arena_handle(kt_ctx* ctx, void* handle64);
KT_API int kt_mgpu_connect(kt_ctx* ctx, const void* handles /* world x 64 bytes */, int world);
KT_API int kt_mgpu_info(kt_ctx* ctx, int* info5);
KT_API int kt_mgpu_export_tsdf_replica(kt_ctx* ctx, int16_t* tsdf_host /* vol^3 */);
KT_API long long kt_launch_count(kt_ctx* ctx);
/* debug: 64 x 5 clock64() stamps of the last whole-frame ICP launch (recorded only while stage timing is enabled) */
KT_API int kt_debug_icp_profile(kt_ctx* ctx, long long* out512);
/* ---- OdometryProvider level (OdometryProvider.h:42-52) ----
 * One call = ICPOdometry / RGBDOdometry::getIncrementalTransformation (ICPOdometry.cpp:68-186, RGBDOdometry.cpp:165-393) for a caller that
 * owns the pose history (Rprev / tprev in, Rcurr / tcurr out, camera-to-volume) and the maps: the model maps vmaps_g_prev / nmaps_g_prev
 * (volume frame) and optionally the current maps (NULL: built from the depth frame by the fused front end), 4 pyramid levels each,
 * device pointers, SoA x 3 like the reference's DeviceArray2D<float>(3 * rows, cols).  The context (kt_create with the odometry mode and
 * the image geometry; its volume is not touched) lends the kernels' scratch and keeps the photometric last / next pyramids between
 * calls; kt_odometry_first_run = RGBDOdometry::firstRun on the first frame.  The 0.3 m jump guard (RGBDOdometry.cpp:383) applies. */
KT_API int kt_odometry_first_run(kt_ctx* ctx, const uint16_t* depth_dev, const uint8_t* rgb_dev);
KT_API int kt_odometry_increment(kt_ctx* ctx, const uint16_t* depth_dev, const uint8_t* rgb_dev, const float* Rprev9, const float* tprev3,
                          const float* const* vmaps_g_prev4, const float* const* nmaps_g_prev4,
                          const float* const* vmaps_curr4, const float* const* nmaps_curr4, float* Rcurr9, float* tcurr3);
/* getLiveImage (KintinuousTracker.cpp:835-862, 960-981, 1125-1154): shaded weight image (uchar3), colour image (uchar3) and model depth
 * (u16 mm) of the surface predicted at the last pose; host buffers of rows*cols pixels, any may be NULL. */
KT_API int kt_get_live_image(kt_ctx* ctx, uint8_t* shaded_rgb_host, uint8_t* color_rgb_host, uint16_t* model_depth_host);
/* getLiveTsdf (.cpp:835-850, 1087-1123): surface points of the whole volume at this moment, without recording a slice.
 * *count = points found (clamped to the cloud buffer capacity); up to max_points are copied. */
KT_API int kt_get_live_tsdf(kt_ctx* ctx, kt_point_xyzrgb* points_host, size_t max_points, size_t* count);
/* debug / parity tap: the arguments of the last integrateTsdfVolume call of the tracker (KintinuousTracker.cpp:864-876): Rcurr^-1
 * (9, row-major), tcurr after the shift adjustment (3), vWrapCopy (3).  Lets a test replay the frame with the reference's own
 * operators on the tracker's own poses and demand a bit-identical volume. */
KT_API int kt_debug_last_integrate(kt_ctx* ctx, float* Rinv9, float* t3, int* wrap3);
KT_API int kt_alloc_pinned(void** ptr, size_t bytes);
KT_API int kt_free_pinned(void* ptr);

/* ---- operators: one per free function of cuda/internal.h:299-536 ----
 * The volume operators (kt_op_init_volume, kt_op_clear_volume, kt_op_integrate, kt_op_raycast, kt_op_extract_slice,
 * kt_op_mesh_volume[_keyed]) take any vol that is a positive multiple of 8 and return KT_ERR_INVALID, before any launch, for every
 * other vol: the clears and the initialisation write whole 16-byte words of a row.  (kt_create asks more: a multiple of 32.) */
KT_API int kt_op_bilateral(const uint16_t* src_dev, uint16_t* dst_dev, int rows, int cols, void* stream);                    /* bilateralFilter (bilateral_pyrdown.cu:333) */
KT_API int kt_op_pyrdown(const uint16_t* src_dev, uint16_t* dst_dev, int src_rows, int src_cols, void* stream);             /* pyrDown (:345) */
KT_API int kt_op_create_vmap(const float* intr4, const uint16_t* depth_dev, float* vmap_dev, int rows, int cols, void* stream);   /* createVMap (maps.cu:123) */
KT_API int kt_op_create_nmap(const float* vmap_dev, float* nmap_dev, int rows, int cols, void* stream);                     /* createNMap (maps.cu:140) */
/* fused createVMap + createNMap for one level (the product's own path) */
KT_API int kt_op_create_maps(const float* intr4, const uint16_t* depth_dev, float* vmap_dev, float* nmap_dev, int rows, int cols, void* stream);
/* The fused front end the tracker runs per frame, on caller buffers (2 launches): bilateralFilter + scaleDepth, then pyrDown x3,
 * createVMap / createNMap x4, the per-pixel colour-integration inputs (cw: view-angle weight, sign = normal invalid; rgbf: float4 RGB)
 * and -- when depth_m4 is not NULL -- shortDepthToMetres (cut-off 6 m), imageBGRToIntensity, pyrDownGaussF / pyrDownUcharGauss x3 and
 * computeDerivativeImages x4 (bilateral_pyrdown.cu:60-420, maps.cu:57-155, tsdf_volume.cu:491-538,601-622).  Every *4 argument is an
 * array of 4 device pointers (pyramid levels); depths4[0] receives the filtered depth.  cw / rgbf / depth_scaled may be NULL. */
KT_API int kt_op_frontend(const uint16_t* depth_raw_dev, const uint8_t* rgb_dev, int rows, int cols, const float* intr4, int angle_color,
                   uint16_t* const* depths4, float* const* vmaps4, float* const* nmaps4, float* depth_scaled_dev, float* cw_dev, float* rgbf_dev,
                   float* const* depth_m4, uint8_t* const* intensity4, int16_t* const* dIdx4, int16_t* const* dIdy4, void* stream);
KT_API int kt_op_transform_maps(const float* vmap_src, const float* nmap_src, const float* R9, const float* t3,
                         float* vmap_dst, float* nmap_dst, int rows, int cols, void* stream);                        /* tranformMaps (maps.cu:204) */
KT_API int kt_op_resize_vmap(const float* in_dev, float* out_dev, int in_rows, int in_cols, void* stream);                  /* resizeVMap (maps.cu:299) */
KT_API int kt_op_resize_nmap(const float* in_dev, float* out_dev, int in_rows, int in_cols, void* stream);                  /* resizeNMap (maps.cu:305) */
/* icpStep (reduce.cu:347-419): one normal-equation build; A_host 36, b_host 6, residual_host 2 floats. */
KT_API int kt_op_icp_step(const float* Rcurr9, const float* tcurr3, const float* vmap_curr, const float* nmap_curr,
                   const float* Rprev_inv9, const float* tprev3, const float* intr4,
                   const float* vmap_g_prev, const float* nmap_g_prev, int rows, int cols,
                   float dist_thres, float angle_thres, float* A_host, float* b_host, float* residual_host, void* stream);
/* integrateTsdfVolume (tsdf_volume.cu:643-674): scaleDepth + tsdf23. tsdf: short[vol^3], color: uchar4[vol^3]. */
KT_API int kt_op_integrate(const uint16_t* depth_raw_dev, int rows, int cols, const float* intr4, const float* volume_size3,
                    const float* Rcurr_inv9, const float* tcurr3, float trunc_dist, int16_t* tsdf_dev, uint8_t* color_dev, int vol,
                    const int* voxel_wrap3, const uint8_t* rgb_dev, const float* nmap_curr_dev, int angle_color,
                    float* depth_scaled_dev, void* stream);
/* raycast (ray_caster.cu:434-471) */
KT_API int kt_op_raycast(const float* intr4, const float* Rcurr9, const float* tcurr3, float trunc_dist, const float* volume_size3,
                  const int16_t* tsdf_dev, int vol, float* vmap_dev, float* nmap_dev, int rows, int cols,
                  const int* voxel_wrap3, uint8_t* vmap_color_dev, const uint8_t* color_dev, void* stream);
/* extractCloudSlice (extract.cu:325-419); *count = points written (<= capacity). Point order is unspecified. */
KT_API int kt_op_extract_slice(const int16_t* tsdf_dev, const float* volume_size3, int vol, kt_point_xyzrgb* out_dev, size_t capacity,
                        const int* voxel_wrap3, const uint8_t* color_dev, int minX, int maxX, int minY, int maxY, int minZ, int maxZ,
                        int subsample, const int* real_voxel_wrap3, size_t* count, void* stream);
/* What CloudSliceProcessor::process does to every slice before the backend sees it (backend/CloudSliceProcessor.cpp:97-162): weight cull
 * (alpha >= weight_cull, -cw, default 8; 0 = off), pcl::VoxelGrid with leaf = the voxel edge, pcl::NormalEstimation with k_search = 20
 * nearest neighbours and the viewpoint at the origin, pcl::concatenateFields -- on the device, on a slice that is still there.
 * points_dev: n extracted points; out_dev: room for `capacity` 48-byte points (n is always enough); *count = processed points, in
 * pcl::VoxelGrid's output order (ascending leaf index).  KT_ERR_INVALID if the leaf grid would exceed INT_MAX cells (PCL skips the
 * filter in that case). */
KT_API int kt_op_process_slice(const kt_point_xyzrgb* points_dev, size_t n, int weight_cull, float leaf, int k_search,
                               kt_point_xyzrgbnormal* out_dev, size_t capacity, size_t* count, void* stream);
/* pcl::VoxelGrid<PointT>::applyFilter (PCL 1.7.2, downsample_all_data, kt_map.cu) over n device points of kind 0 (kt_point_xyzrgb) or
 * 1 (kt_point_xyzrgbnormal): one centroid per occupied leaf of edge `leaf`, in ascending leaf index, every field averaged in PCL's float
 * arithmetic (points of a leaf added in input order, from the first point on), colour truncated, alpha 0.  Writes up to `capacity`
 * points of the same kind to out_dev and returns the full count.  Leaf indices are 64-bit: where PCL's int64 check finds more than
 * INT_MAX cells, PCL returns the cloud unfiltered; this filters and sets *pcl_would_skip = 1.  KT_ERR_INVALID for a non-finite x / y / z,
 * more than 2^62 cells or 2^31 - 1 points; KT_ERR_CUDA when its scratch cannot be allocated. */
KT_API int kt_op_voxel_grid(const void* points_dev, size_t n, int kind, float leaf, void* out_dev, size_t capacity, size_t* count,
                            int* pcl_would_skip, void* stream);
/* Marching cubes over the cells of the logical box [minX,maxX) x [minY,maxY) x [minZ,maxZ) of the cyclic volume, with extractCloudSlice's
 * addressing (voxel_wrap3: storage offset, any value, reduced mod vol; real_voxel_wrap3: global offset of the positions).  Stands in
 * for calculateMesh (backend/MeshGenerator.cpp:193-227; a different algorithm, no parity with PCL's greedy projection).  A corner is
 * valid when extractCloudSlice would use it (W != 0, F != 1) and W >= weight_cull; inside when its raw TSDF is < 0.  A cell (lower corner
 * in the box, upper corner < vol on every axis, no cyclic wrap) is meshed when its 8 corners are valid and not all on one side.  Output
 * (device): one vertex per crossing edge of a meshed cell, at exactly the point extractCloudSlice emits for that edge, ordered by the
 * edge's lower voxel (x fastest) then axis; triangles as uint32 triples, ordered by cell then case-table order, (v1-v0)x(v2-v0) pointing
 * to free space.  Deterministic, independent of the launch and of voxel_wrap3.  The counts are always returned; if either output is
 * too small the call returns KT_ERR_CAPACITY and writes neither. */
KT_API int kt_op_mesh_volume(const int16_t* tsdf_dev, const uint8_t* color_dev, int vol, const float* volume_size3,
                             const int* voxel_wrap3, const int* real_voxel_wrap3, int minX, int maxX, int minY, int maxY, int minZ, int maxZ,
                             int weight_cull, kt_mesh_vertex* verts_dev, size_t max_verts, uint32_t* tris_dev, size_t max_tris,
                             size_t* n_verts, size_t* n_tris, void* stream);
/* kt_op_mesh_volume that also says where each vertex and triangle is on the global voxel lattice: vert_edges_dev gets (gx, gy, gz, axis)
 * per vertex, the lower voxel and axis of its edge, and tri_cells_dev (gx, gy, gz, 0) per triangle, the lower corner of its cell, both
 * int32 x 4 and global = logical voxel + real_voxel_wrap3.  Vertices and triangles are byte-identical to kt_op_mesh_volume's, with the
 * same capacity contract (max_verts bounds vert_edges_dev too, max_tris tri_cells_dev). */
KT_API int kt_op_mesh_volume_keyed(const int16_t* tsdf_dev, const uint8_t* color_dev, int vol, const float* volume_size3,
                                   const int* voxel_wrap3, const int* real_voxel_wrap3, int minX, int maxX, int minY, int maxY, int minZ, int maxZ,
                                   int weight_cull, kt_mesh_vertex* verts_dev, int32_t* vert_edges_dev, size_t max_verts, uint32_t* tris_dev,
                                   int32_t* tri_cells_dev, size_t max_tris, size_t* n_verts, size_t* n_tris, void* stream);
/* Marching cubes over a sparse set of 8^3 bricks (device): keys strictly ascending (kt_set_map_volume's key layout), 512 int16 tsdf and
 * 512 x 4 uint8 colour per brick.  kt_op_mesh_volume's contract with the global voxel as the logical one and no border: a voxel outside
 * every brick is unobserved.  Positions as kt_op_mesh_volume's with real_voxel_wrap 0 and this vol (cell = volume_size3 / vol); the
 * order is kt_get_global_mesh's.  NULL outputs: counts only; KT_ERR_CAPACITY (nothing written) when they exceed the capacities;
 * KT_ERR_INVALID for unsorted keys.  Synchronous. */
KT_API int kt_op_mesh_bricks(const uint64_t* keys_dev, const int16_t* tsdf_dev, const uint8_t* color_dev, size_t n_bricks, const float* volume_size3,
                             int vol, int weight_cull, kt_mesh_vertex* verts_dev, size_t max_verts, uint32_t* tris_dev, size_t max_tris,
                             size_t* n_verts, size_t* n_tris, void* stream);
/* Weld n_meshes keyed meshes (kt_op_mesh_volume_keyed, kt_get_slice_mesh_keys) into one (kt_weld.cu).  Input (device): the meshes
 * concatenated in order -- vertices with their edges, triangles (indices local to their own mesh) with their cells -- and n_meshes + 1
 * HOST offsets of each mesh's first vertex / triangle (vert_offsets_host[n_meshes] = all vertices).
 *   - Cell winner: every global cell keeps the triangles of the highest-numbered mesh that has triangles there; a cell only one mesh
 *     meshed keeps that mesh's.
 *   - Vertex weld: only vertices a kept triangle uses are kept; of those on one global edge, the highest-numbered mesh's (32 bytes
 *     copied unchanged) represents them all.
 *   - Order: vertices ascend by (gz, gy, gx, axis), triangles by cell (gz, gy, gx) and within a cell in the winning mesh's order; indices
 *     point into the output.  This is kt_op_mesh_volume's order, so welding keyed meshes of overlapping boxes of one volume gives exactly
 *     the union box's mesh.  Deterministic: two calls give byte-identical output.
 * No triangles in: nothing out.  KT_ERR_INVALID for n_meshes < 1, null or descending offsets, more than 2^31 - 1 vertices or triangles
 * in, an axis outside 0..2, an index outside its mesh, or keys beyond 2^62 (3 x the voxels of the lattice box the keys span);
 * KT_ERR_CAPACITY when either output is too small (both counts returned, nothing written); KT_ERR_CUDA when its scratch cannot be
 * allocated.  report (may be NULL): the counts, sort_ms /
 * weld_ms / total_ms. */
KT_API int kt_op_weld_meshes(const kt_mesh_vertex* verts_dev, const int32_t* vert_edges_dev, const size_t* vert_offsets_host,
                             const uint32_t* tris_dev, const int32_t* tri_cells_dev, const size_t* tri_offsets_host, int n_meshes,
                             kt_mesh_vertex* out_verts_dev, size_t max_verts, uint32_t* out_tris_dev, size_t max_tris, size_t* n_verts, size_t* n_tris,
                             kt_weld_report* report, void* stream);
/* Deformation graph operators (kt_deform_map runs the three in turn).  Nodes: n_nodes float xyz positions and their uint64 times,
 * ascending (device).  kind: 0 = kt_point_xyzrgbnormal, 1 = kt_mesh_vertex, 2 = packed float xyz (weights only).
 * kt_op_deform_weights -- weightVerticesSeq (DeformationGraph.cpp:441-556): per point, the node nearest its time by binary search (a time
 * outside the node times clamps to the first / last node; the reference reads past both ends there), the 20 consecutive candidates from
 * it (back, topped up forward), the k+1 = 5 nearest (float distances, ties by id), weights (1 - |v - g_j| / dMax)^2 in FP64 for the 4
 * nearest, normalised; out: 4 int32 node ids ascending and their 4 FP64 weights per point.  Fewer than 5 nodes: KT_ERR_STATE. */
KT_API int kt_op_deform_weights(const float* node_pos_dev, const uint64_t* node_times_dev, int n_nodes, const void* points_dev, int kind,
                                const uint64_t* times_dev, size_t n, int32_t* ids_dev, double* weights_dev, void* stream);
/* optimiseGraphSparse (DeformationGraph.cpp:714-774) over the sequentially connected nodes (connectGraphSeq :217-271, k = 4) with one
 * position constraint per row of con_src (float xyz, device) -> con_dst (double xyz, device), weighted by kt_op_deform_weights' output
 * for the sources.  Out: 12 doubles per node (rotation column-major, then translation; the identity when report->deformed is 0) and the
 * report.  The normal equations are solved on the device by a block-banded Cholesky; a term spanning more than 19 node blocks returns
 * KT_ERR_INVALID. */
KT_API int kt_op_deform_optimise(const float* node_pos_dev, int n_nodes, const float* con_src_dev, const double* con_dst_dev,
                                 const int32_t* con_ids_dev, const double* con_weights_dev, size_t n_con, double* params_dev,
                                 kt_deform_report* report, void* stream);
/* applyGraphToVertices / computeVertexPosition (DeformationGraph.cpp:644-677, :1028-1054): kind 0 or 1 records from in_dev to out_dev,
 * position sum_j w_j (R_j (v - g_j) + g_j + t_j), normal sum_j w_j R_j^-T n normalised (zero stays zero), FP64 written as float, every
 * other byte copied. */
KT_API int kt_op_deform_apply(const float* node_pos_dev, const double* params_dev, int n_nodes, const int32_t* ids_dev,
                              const double* weights_dev, const void* in_dev, void* out_dev, int kind, size_t n, void* stream);
/* Pose-graph optimisation (isam::Slam::batch_optimization as kt_close_loop runs it).  poses_dev: n_nodes 4 x 4 row-major FP64 node
 * poses, the initial estimate; factors_dev: n_factors kt_pgo_factor records -- factor 0 the prior on node 0 (i = -1, z = the anchor's
 * Pose3d vector x y z yaw pitch roll), factor k (1 <= k < n_nodes) odometry k-1 -> k, then at most 64 loops (any i != j); z of a
 * between factor is the measured (p_j (-) p_i).vector().  out_dev: the optimised poses (may equal poses_dev).  Any other list shape:
 * KT_ERR_INVALID; more than 2^18 nodes or 64 loops: KT_ERR_CAPACITY. */
typedef struct kt_pgo_factor { int32_t i, j; double z[6]; } kt_pgo_factor;
typedef struct kt_pgo_report {
    int nodes, factors, loops, iterations;
    double chi2_initial, chi2_final;
    int solver_failed;
    double step_ms;                 /* mean device time of a Gauss-Newton step (assembly to the chi2 of the updated poses), CUDA events */
} kt_pgo_report;
KT_API int kt_op_pgo_optimise(const double* poses_dev, int n_nodes, const kt_pgo_factor* factors_dev, int n_factors, double* out_dev,
                              kt_pgo_report* report, void* stream);
/* ---- place-recognition operators (what kt_detect_loops runs; device pointers) ----
 * kt_op_surf -- cv::SURF(400, 4, 2, false) on the grey image (PlaceRecognition.cpp:51-88, DBowInterfaceSurf.cpp:72-99), restated from
 * Bay et al. 2008 (kt_surf.cu header): rgb rows*cols*3 -> at most max_features keypoints, strongest first (ties by octave, layer,
 * position), kp 6 floats each (x, y, size, angle in radians, response, laplacian sign), desc 64 floats each; *n_out (host). */
KT_API int kt_op_surf(const uint8_t* rgb_dev, int rows, int cols, float hessian_threshold, int max_features, float* kp_dev, float* desc_dev,
                      int* n_out, void* stream);
/* kt_op_keypoints_3d -- Surf3DTools::calculate3dPointsSURF's lookup (Surf3DTools.h:82, :142-160), what kt_detect_loops runs on every
 * keyframe's keypoints: kp n x 6 floats (kt_op_surf's layout, x and y used), depth rows*cols u16 mm, both device; xyz n x 3 floats
 * (device) in the depth camera, NaN for a keypoint without a point (not within +-0.5 px of a pixel, strict, depth 0, or z >= 10 m). */
KT_API int kt_op_keypoints_3d(const float* kp_dev, int n, const uint16_t* depth_dev, int rows, int cols, const float* intr4, float* xyz_dev,
                              void* stream);
/* kt_op_match_ratio -- the ratio test of Surf3DTools::surfMatch3D (Surf3DTools.h:105-140) with an exact 2-NN in place of FLANN, and the
 * retrieval kt_detect_loops runs with it: the database is n_seg segments (keyframes) of `stride` rows of 64 floats, of which the first
 * seg_counts[g] are valid (host array; NULL: all).  For each valid row the two nearest of n_query query descriptors (squared distances),
 * best index and pass = d1 < ratio d2 (an invalid row: best -1, pass 0); seg_passes (host, n_seg ints, may be NULL): passes per segment. */
KT_API int kt_op_match_ratio(const float* db_dev, int n_seg, int stride, const int* seg_counts, const float* query_dev, int n_query, float ratio,
                             int* best_dev, float* d1_dev, float* d2_dev, uint8_t* pass_dev, int* seg_passes, void* stream);
/* kt_op_pnp_ransac -- PNPSolver::getRelativePose / cv::solvePnPRansac (PNPSolver.cpp:51-75): n matches of new-camera xyz (p_new) with
 * old-camera xyz (p_old) and old-image pixels (uv_old), host arrays.  pose12 (host): R row-major and t of p_old ~ R p_new + t; inliers
 * (host, n bytes); *n_inliers. */
KT_API int kt_op_pnp_ransac(const float* p_new, const float* p_old, const float* uv_old, int n, const float* intr4, int iterations,
                            float threshold_px, uint64_t seed, double* pose12, uint8_t* inliers, int* n_inliers);
/* kt_op_cloud_fitness -- IterativeClosestPoint::getFitnessScore after PlaceRecognition::icpDepthFrames (PlaceRecognition.cpp:238-276):
 * both depth images (device, u16 mm) as clouds, voxel-grid filtered at leaf, source moved by T12 (3 x 4 row-major, host), mean squared
 * distance to the nearest target point. */
KT_API int kt_op_cloud_fitness(const uint16_t* src_depth_dev, const uint16_t* dst_depth_dev, int rows, int cols, const float* intr4, float leaf,
                               const float* T12, double* fitness, size_t* n_src, size_t* n_dst);
/* clearVolume{X,Y,Z}[Back] + ...c on both volumes (tsdf_volume.cu:117-448). axis 0..2, back 0/1. */
KT_API int kt_op_clear_volume(int axis, int back, int16_t* tsdf_dev, uint8_t* color_dev, int vol, int current_wrap, int delta_wrap, void* stream);
/* initVolume + initColorVolume (tsdf_volume.cu:469, :77) */
KT_API int kt_op_init_volume(int16_t* tsdf_dev, uint8_t* color_dev, int vol, void* stream);
/* RGB-D odometry operators (bilateral_pyrdown.cu:300-420, maps.cu:331, reduce.cu:555,798) */
KT_API int kt_op_short_depth_to_metres(const uint16_t* src_dev, float* dst_dev, int rows, int cols, int cut_off, void* stream);
KT_API int kt_op_pyrdown_gauss_f(const float* src_dev, float* dst_dev, int src_rows, int src_cols, void* stream);
KT_API int kt_op_bgr_to_intensity(const uint8_t* rgb_dev, uint8_t* dst_dev, int rows, int cols, void* stream);
KT_API int kt_op_pyrdown_uchar_gauss(const uint8_t* src_dev, uint8_t* dst_dev, int src_rows, int src_cols, void* stream);
KT_API int kt_op_derivative_images(const uint8_t* src_dev, int16_t* dx_dev, int16_t* dy_dev, int rows, int cols, void* stream);
KT_API int kt_op_project_to_point_cloud(const float* depth_dev, float* cloud_dev, int rows, int cols, const double* intr4, int level, void* stream);
KT_API int kt_op_rgb_residual(float min_scale, const int16_t* dIdx, const int16_t* dIdy, const float* last_depth, const float* next_depth,
                       const uint8_t* last_image, const uint8_t* next_image, void* corres_dev, int rows, int cols,
                       float max_depth_delta, const float* kt3, const float* krkinv9, int* sigma_sum, int* count, void* stream);
KT_API int kt_op_rgb_step(const void* corres_dev, float sigma, const float* cloud_dev, float fx, float fy, const int16_t* dIdx, const int16_t* dIdy,
                   float sobel_scale, int rows, int cols, float* A_host, float* b_host, void* stream);

/* generateImage (image_generator.cu:161-186): shaded weight heat-map image (dst) and colour image (dstColor) of the predicted surface,
 * uchar3 each, either may be NULL; light = LightSource {pos[1], number}.  generateDepth (:187-230): model depth in mm from the model
 * vertex map, row 3 of R^-1 and t (max_depth is unused there as well). */
KT_API int kt_op_generate_image(const float* vmap_dev, const float* nmap_dev, const uint8_t* vmap_curr_color_dev, const float* light_pos3, int n_lights,
                         uint8_t* dst_rgb_dev, uint8_t* dst_color_rgb_dev, int rows, int cols, void* stream);
KT_API int kt_op_generate_depth(const float* Rcurr_inv9, const float* tcurr3, const float* vmap_dev, const float* nmap_dev, uint16_t* dst_dev,
                         int rows, int cols, float max_depth, void* stream);

/* ---- .klg log reader: replaces RawLogReader (src/utils/RawLogReader.cpp:20-133) and the upload + processFrame body of
 * TrackerInterface::process (src/backend/TrackerInterface.cpp:82-104).  File layout: int32 numFrames, then per frame int64 timestamp,
 * int32 depthSize, int32 imageSize, depth bytes (zlib stream or raw u16), image bytes (JPEG, raw 24-bit, or none).  Depth is inflated
 * into pinned memory and copied asynchronously; a JPEG is decoded ON THE DEVICE (nvJPEG) into the interleaved B,G,R bytes cvDecodeImage
 * produces.  The pointers of a frame stay valid until the next-but-one kt_klg_read_next. ---- */
typedef struct kt_klg kt_klg;
typedef struct kt_klg_frame {
    int64_t timestamp;                 /* RawLogReader::timestamp */
    int32_t depth_size, image_size;    /* compressedDepthSize / compressedImageSize */
    int is_compressed;                 /* RawLogReader::isCompressed */
    int frame;                         /* currentFrame after the read */
    const uint16_t* depth_dev;         /* rows*cols u16, device (valid after kt_klg_wait) */
    const uint8_t* rgb_dev;            /* rows*cols*3 u8, device */
    const uint16_t* depth_host;        /* decompressedDepth, pinned host memory */
    const unsigned char* compressed_depth; const unsigned char* compressed_image;   /* the frame's stored bytes (place-recognition inputs of processFrame) */
} kt_klg_frame;
KT_API int kt_klg_open(const char* path, int rows, int cols, int device, kt_klg** out);   /* RawLogReader::RawLogReader (:20-41) */
KT_API int kt_klg_close(kt_klg* log);                                                     /* ~RawLogReader (:43-49) */
KT_API int kt_klg_num_frames(kt_klg* log);                                                /* numFrames */
KT_API int kt_klg_has_more(kt_klg* log);                                                  /* hasMore */
KT_API int kt_klg_set_flip_colors(kt_klg* log, int flip);                                 /* ConfigArgs::flipColors (-f), :117-125 */
KT_API int kt_klg_read_next(kt_klg* log, kt_klg_frame* out);                              /* readNext (:52-133); transfers are in flight on return */
KT_API int kt_klg_wait(kt_klg* log);                                                      /* the last frame read has landed on the device */
KT_API int kt_klg_track_next(kt_klg* log, kt_ctx* ctx, kt_pose* out);                     /* TrackerInterface::process (:82-104): read, upload, processFrame */

#ifdef __cplusplus
}
#endif
#endif /* KINTINUOUS_B200_H_ */
