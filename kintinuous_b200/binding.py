"""ctypes binding of include/kintinuous_b200.h (the drop-in C ABI)."""
from __future__ import annotations

import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class KtError(RuntimeError):
    pass


def lib_path() -> str:
    return os.path.join(_HERE, "libkintinuous_b200.so")


def load():
    """Load the CUDA library; raises (loudly) if it was not built -- there is no fallback path."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not os.path.exists(p):
        raise KtError(f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                      f"(or make -C kintinuous_b200/csrc); kintinuous_b200 has no CPU fallback")
    lib = C.CDLL(p)
    lib.kt_last_error.restype = C.c_char_p
    lib.kt_get_voxel_size.restype = C.c_float
    lib.kt_get_trunc_dist.restype = C.c_float
    lib.kt_launch_count.restype = C.c_longlong
    lib.kt_get_icp_kernel_ms.restype = C.c_float
    lib.kt_span_elapsed_ms.restype = C.c_float
    _LIB = lib
    return lib


def cuda_available() -> bool:
    return bool(load().kt_cuda_available())


def _check(status: int):
    if status != 0:
        raise KtError(f"kintinuous_b200 error {status}: {load().kt_last_error().decode()}")


class Config(C.Structure):
    """kt_config (include/kintinuous_b200.h)."""
    _fields_ = [("rows", C.c_int), ("cols", C.c_int),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("vol", C.c_int), ("volume_size", C.c_float),
                ("odometry", C.c_int), ("fast_odometry", C.c_int), ("voxel_shift", C.c_int), ("overlap", C.c_int),
                ("angle_color", C.c_int), ("parked", C.c_int), ("cloud_capacity", C.c_int), ("device", C.c_int),
                ("rank", C.c_int), ("world", C.c_int)]

    @staticmethod
    def default(rows=480, cols=640, vol=512, volume_size=6.0, odometry=0, **kw):
        from . import synth
        fx, fy, cx, cy = synth.intrinsics(cols, rows)
        c = Config(rows=rows, cols=cols, fx=fx, fy=fy, cx=cx, cy=cy, vol=vol, volume_size=volume_size, odometry=odometry,
                   fast_odometry=0, voxel_shift=14, overlap=2, angle_color=1, parked=0, cloud_capacity=0, device=0, rank=0, world=1)
        for k, v in kw.items():
            setattr(c, k, v)
        return c


class DensePose(C.Structure):
    _fields_ = [("timestamp", C.c_uint64), ("pose", C.c_float * 16), ("is_loop_pose", C.c_int)]


class DeformConstraint(C.Structure):
    """kt_deform_constraint: a point that belongs elsewhere (time, position in the map as tracked, target)."""
    _fields_ = [("time", C.c_uint64), ("source", C.c_float * 3), ("target", C.c_float * 3)]


class DeformReport(C.Structure):
    """kt_deform_report of kt_deform_map / kt_op_deform_optimise."""
    _fields_ = [("nodes", C.c_int), ("constraints", C.c_int), ("band", C.c_int), ("iterations", C.c_int),
                ("initial_error", C.c_double), ("final_error", C.c_double), ("constraint_error", C.c_double),
                ("deformed", C.c_int), ("solver_failed", C.c_int)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class LoopConstraint(C.Structure):
    """kt_loop_constraint: PlaceRecognition's LoopClosureConstraint (time1 new, time2 old, pose of time2 in time1's camera, inliers)."""
    _fields_ = [("time1", C.c_uint64), ("time2", C.c_uint64), ("constraint", C.c_double * 16), ("inliers1", C.c_void_p),
                ("inliers2", C.c_void_p), ("n_inliers", C.c_size_t)]


class LoopReport(C.Structure):
    """kt_loop_report of kt_close_loop."""
    _fields_ = [("nodes", C.c_int), ("factors", C.c_int), ("loops", C.c_int), ("iterations", C.c_int),
                ("chi2_initial", C.c_double), ("chi2_final", C.c_double), ("accepted", C.c_int), ("solver_failed", C.c_int),
                ("map_deformed", C.c_int), ("deform", DeformReport)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k != "deform"}
        d["deform"] = self.deform.as_dict()
        return d


class LoopDetectionParams(C.Structure):
    """kt_loop_detection_params (kt_default_loop_detection gives the reference's defaults)."""
    _fields_ = [("enabled", C.c_int), ("inlier_ratio", C.c_float), ("loop_throttle_s", C.c_double), ("isam_thresh", C.c_double),
                ("node_spacing", C.c_float), ("pose_spacing", C.c_float), ("max_keyframes", C.c_int), ("max_features", C.c_int),
                ("exclude_recent", C.c_int), ("close", C.c_int)]


class PlaceResult(C.Structure):
    """kt_place_result of kt_detect_loops: one per keyframe processed."""
    _fields_ = [("keyframe", C.c_int), ("time", C.c_uint64), ("candidate", C.c_int), ("candidate_time", C.c_uint64), ("passes", C.c_int),
                ("matches", C.c_int), ("inliers", C.c_int), ("inlier_ratio", C.c_float), ("fitness", C.c_double), ("stage", C.c_int),
                ("constraint", LoopConstraint), ("closed", C.c_int), ("report", LoopReport)]

    STAGES = ("loop", "throttled", "no_candidate", "matches", "inliers", "fitness")

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k not in ("constraint", "report")}
        d["stage_name"] = self.STAGES[self.stage]
        d["constraint"] = np.array(self.constraint.constraint, np.float64).reshape(4, 4)
        n = int(self.constraint.n_inliers)
        if n:
            d["inliers1"] = np.ctypeslib.as_array(C.cast(self.constraint.inliers1, C.POINTER(C.c_float)), shape=(n * 3,)).reshape(n, 3).copy()
            d["inliers2"] = np.ctypeslib.as_array(C.cast(self.constraint.inliers2, C.POINTER(C.c_float)), shape=(n * 3,)).reshape(n, 3).copy()
        else:
            d["inliers1"] = d["inliers2"] = np.zeros((0, 3), np.float32)
        d["report"] = self.report.as_dict()
        return d


class PgoReport(C.Structure):
    """kt_pgo_report of kt_op_pgo_optimise."""
    _fields_ = [("nodes", C.c_int), ("factors", C.c_int), ("loops", C.c_int), ("iterations", C.c_int),
                ("chi2_initial", C.c_double), ("chi2_final", C.c_double), ("solver_failed", C.c_int), ("step_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# kt_pgo_factor (56 bytes): i = -1 for the prior on node j
PGO_FACTOR_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("z", "<f8", (6,))])
assert PGO_FACTOR_DTYPE.itemsize == 56


class MapReport(C.Structure):
    """kt_map_report of kt_get_map_cloud / kt_save_map_pcd."""
    _fields_ = [("input_points", C.c_size_t), ("output_points", C.c_size_t), ("slices", C.c_int), ("moved_slices", C.c_int),
                ("pcl_would_skip", C.c_int), ("upload_ms", C.c_float), ("sort_ms", C.c_float), ("centroid_ms", C.c_float),
                ("download_ms", C.c_float), ("total_ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class WeldReport(C.Structure):
    """kt_weld_report of kt_get_map_mesh / kt_save_map_ply / kt_op_weld_meshes."""
    _fields_ = [("input_verts", C.c_size_t), ("input_tris", C.c_size_t), ("output_verts", C.c_size_t), ("output_tris", C.c_size_t),
                ("repeated_cells", C.c_size_t), ("dropped_triangles", C.c_size_t), ("merged_vertices", C.c_size_t), ("meshes", C.c_int),
                ("moved_meshes", C.c_int), ("upload_ms", C.c_float), ("sort_ms", C.c_float), ("weld_ms", C.c_float),
                ("download_ms", C.c_float), ("total_ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class GlobalMeshReport(C.Structure):
    """kt_global_mesh_report of kt_get_global_mesh / kt_save_global_mesh_ply."""
    _fields_ = [("bricks", C.c_size_t), ("store_bricks", C.c_size_t), ("live_bricks", C.c_size_t), ("input_voxels", C.c_size_t),
                ("output_verts", C.c_size_t), ("output_tris", C.c_size_t), ("store_full", C.c_int), ("gather_ms", C.c_float),
                ("mesh_ms", C.c_float), ("sort_ms", C.c_float), ("download_ms", C.c_float), ("total_ms", C.c_float)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class SliceInfo(C.Structure):
    _fields_ = [("dimension", C.c_int), ("odometry", C.c_int), ("camera_t", C.c_float * 3), ("camera_R", C.c_float * 9),
                ("utime", C.c_uint64), ("count", C.c_size_t)]


class Pose(C.Structure):
    _fields_ = [("R", C.c_float * 9), ("t", C.c_float * 3), ("global_t", C.c_float * 3), ("voxel_wrap", C.c_int * 3),
                ("shifted", C.c_int), ("frame", C.c_int)]

    def as_tuple(self):
        return (np.array(self.R, dtype=np.float32).reshape(3, 3), np.array(self.t, dtype=np.float32),
                np.array(self.global_t, dtype=np.float32), np.array(self.voxel_wrap, dtype=np.int32))


POINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("_p0", "<f4"),
                        ("b", "u1"), ("g", "u1"), ("r", "u1"), ("a", "u1"), ("_p1", "u1", (12,))])
assert POINT_DTYPE.itemsize == 32
# kt_point_xyzrgbnormal == pcl::PointXYZRGBNormal (48 bytes)
POINT_NORMAL_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("_p0", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"), ("_p1", "<f4"),
                               ("b", "u1"), ("g", "u1"), ("r", "u1"), ("a", "u1"), ("curvature", "<f4"), ("_p2", "<f4", (2,))])
assert POINT_NORMAL_DTYPE.itemsize == 48
# kt_mesh_vertex (32 bytes): position, unit normal, colour, alpha = weight
MESH_VERTEX_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                              ("r", "u1"), ("g", "u1"), ("b", "u1"), ("a", "u1"), ("_pad", "<u4")])
assert MESH_VERTEX_DTYPE.itemsize == 32
KT_ERR_CAPACITY = -4


def _ptr(a):
    """Device pointer of a torch tensor / int, host pointer of a numpy array."""
    if a is None:
        return C.c_void_p(0)
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(a.data_ptr())


def _f(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(-1))


class Tracker:
    """Mirror of the reference's KintinuousTracker (KintinuousTracker.h:85-172) over the C ABI."""

    def __init__(self, cfg: Config):
        self.lib = load()
        self.cfg = cfg
        self.h = C.c_void_p()
        _check(self.lib.kt_create(C.byref(cfg), C.byref(self.h)))

    def close(self):
        if self.h:
            self.lib.kt_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        _check(self.lib.kt_reset(self.h))

    def process_frame(self, depth: np.ndarray, rgb: np.ndarray, utime: int = 0) -> Pose:
        """processFrame with HOST buffers (numpy, or raw pinned pointers as ints)."""
        p = Pose()
        _check(self.lib.kt_process_frame(self.h, _ptr(depth), _ptr(rgb), C.c_uint64(utime), C.byref(p)))
        return p

    def prefetch_frame(self, depth, rgb):
        """Hint: start the H2D copy of the next frame now (kt_prefetch_frame)."""
        _check(self.lib.kt_prefetch_frame(self.h, _ptr(depth), _ptr(rgb)))

    def process_frame_device(self, depth_dev, rgb_dev, utime: int = 0) -> Pose:
        p = Pose()
        _check(self.lib.kt_process_frame_device(self.h, _ptr(depth_dev), _ptr(rgb_dev), C.c_uint64(utime), C.byref(p)))
        return p

    def finalise(self):
        _check(self.lib.kt_finalise(self.h))

    def pose(self) -> Pose:
        p = Pose()
        _check(self.lib.kt_get_pose(self.h, C.byref(p)))
        return p

    @property
    def voxel_size(self):
        return float(self.lib.kt_get_voxel_size(self.h))

    @property
    def trunc_dist(self):
        return float(self.lib.kt_get_trunc_dist(self.h))

    def num_slices(self):
        return int(self.lib.kt_num_slices(self.h))

    def get_slice(self, idx):
        n = C.c_size_t(0); dim = C.c_int(0); cam = (C.c_float * 3)()
        _check(self.lib.kt_get_slice(self.h, idx, None, C.c_size_t(0), C.byref(n), C.byref(dim), cam))
        pts = np.zeros(n.value, dtype=POINT_DTYPE)
        if n.value:
            _check(self.lib.kt_get_slice(self.h, idx, _ptr(pts), C.c_size_t(n.value), C.byref(n), C.byref(dim), cam))
        return pts, dim.value, np.array(cam, dtype=np.float32)

    def num_dense_poses(self):
        return int(self.lib.kt_num_dense_poses(self.h))

    def dense_pose(self, idx):
        """(timestamp, 4x4 pose [R | currentGlobalCamera], is_loop_pose) of densePoseGraph[idx]."""
        d = DensePose()
        _check(self.lib.kt_get_dense_pose(self.h, idx, C.byref(d)))
        return int(d.timestamp), np.array(d.pose, np.float32).reshape(4, 4), bool(d.is_loop_pose)

    def set_pose_log(self, path):
        _check(self.lib.kt_set_pose_log(self.h, path.encode() if path else None))

    def set_slice_processing(self, enabled=True, weight_cull=8):
        """CloudSliceProcessor on the device for every slice recorded from now on (kt_set_slice_processing)."""
        _check(self.lib.kt_set_slice_processing(self.h, int(enabled), int(weight_cull)))

    def get_processed_slice(self, idx):
        n = C.c_size_t(0)
        _check(self.lib.kt_get_processed_slice(self.h, idx, None, C.c_size_t(0), C.byref(n)))
        pts = np.zeros(n.value, dtype=POINT_NORMAL_DTYPE)
        if n.value:
            _check(self.lib.kt_get_processed_slice(self.h, idx, _ptr(pts), C.c_size_t(n.value), C.byref(n)))
        return pts

    def set_slice_meshing(self, enabled=True, weight_cull=8):
        """Marching-cubes mesh of every slice recorded from now on (kt_set_slice_meshing)."""
        _check(self.lib.kt_set_slice_meshing(self.h, int(enabled), int(weight_cull)))

    def get_slice_mesh(self, idx):
        """(vertices MESH_VERTEX_DTYPE [n], triangles uint32 [m, 3]) of slice idx."""
        nv = C.c_size_t(0); nt = C.c_size_t(0)
        _check(self.lib.kt_get_slice_mesh(self.h, idx, None, C.c_size_t(0), None, C.c_size_t(0), C.byref(nv), C.byref(nt)))
        v = np.zeros(nv.value, MESH_VERTEX_DTYPE); t = np.zeros((nt.value, 3), np.uint32)
        _check(self.lib.kt_get_slice_mesh(self.h, idx, _ptr(v), C.c_size_t(len(v)), _ptr(t), C.c_size_t(len(t)), C.byref(nv), C.byref(nt)))
        return v, t

    def get_slice_mesh_keys(self, idx):
        """(vertex edges int32 [n, 4] = gx, gy, gz, axis; triangle cells int32 [m, 4] = gx, gy, gz, 0) of slice idx's mesh on the global
        voxel lattice (kt_get_slice_mesh_keys)."""
        nv = C.c_size_t(0); nt = C.c_size_t(0)
        _check(self.lib.kt_get_slice_mesh(self.h, idx, None, C.c_size_t(0), None, C.c_size_t(0), C.byref(nv), C.byref(nt)))
        e = np.zeros((nv.value, 4), np.int32); k = np.zeros((nt.value, 4), np.int32)
        _check(self.lib.kt_get_slice_mesh_keys(self.h, idx, _ptr(e), C.c_size_t(len(e)), _ptr(k), C.c_size_t(len(k))))
        return e, k

    def map_mesh(self, which=0, weld=True):
        """The map as one mesh (kt_get_map_mesh): which 0 = the recorded map, 1 = the corrected map; weld = every global cell and edge
        once (the latest slice wins), else the slice meshes concatenated.  Returns (MESH_VERTEX_DTYPE [n], uint32 [m, 3], report dict).
        Counts first, then fetches: that runs the export twice."""
        nv = C.c_size_t(0); nt = C.c_size_t(0); rep = WeldReport()
        _check(self.lib.kt_get_map_mesh(self.h, int(which), int(weld), None, C.c_size_t(0), None, C.c_size_t(0), C.byref(nv), C.byref(nt), C.byref(rep)))
        v = np.zeros(nv.value, MESH_VERTEX_DTYPE); t = np.zeros((nt.value, 3), np.uint32)
        if nv.value or nt.value:
            _check(self.lib.kt_get_map_mesh(self.h, int(which), int(weld), _ptr(v), C.c_size_t(len(v)), _ptr(t), C.c_size_t(len(t)),
                                            C.byref(nv), C.byref(nt), C.byref(rep)))
        assert (nv.value, nt.value) == (len(v), len(t))
        return v, t, rep.as_dict()

    def save_map_ply(self, path, which=0, weld=True):
        """The same mesh as a binary PLY in save_mesh_ply's layout (kt_save_map_ply).  Returns the report dict."""
        rep = WeldReport()
        _check(self.lib.kt_save_map_ply(self.h, os.fsencode(path), int(which), int(weld), C.byref(rep)))
        return rep.as_dict()

    def set_map_volume(self, enabled=True, max_bricks=1 << 16):
        """The map volume (kt_set_map_volume): a sparse global TSDF of every voxel a shift clears, in 8^3 bricks; 0 frees it."""
        _check(self.lib.kt_set_map_volume(self.h, int(enabled), C.c_size_t(max_bricks)))

    def set_map_volume_restore(self, enabled=True):
        """Refill the planes each shift clears from the map volume (kt_set_map_volume_restore); needs the map volume on."""
        _check(self.lib.kt_set_map_volume_restore(self.h, int(enabled)))

    def map_volume_info(self):
        """(bricks stored, capacity, full) of the map volume."""
        b = C.c_size_t(0); cap = C.c_size_t(0); full = C.c_int(0)
        _check(self.lib.kt_get_map_volume_info(self.h, C.byref(b), C.byref(cap), C.byref(full)))
        return b.value, cap.value, bool(full.value)

    def map_volume_bricks(self):
        """The stored bricks sorted by key: (keys uint64 [n], tsdf int16 [n, 8, 8, 8], colour uint8 [n, 8, 8, 8, 4]), voxels indexed [z, y, x]."""
        n = C.c_size_t(0)
        _check(self.lib.kt_get_map_volume_bricks(self.h, None, None, None, C.c_size_t(0), C.byref(n)))
        k = np.zeros(n.value, np.uint64); t = np.zeros((n.value, 8, 8, 8), np.int16); c = np.zeros((n.value, 8, 8, 8, 4), np.uint8)
        if n.value:
            _check(self.lib.kt_get_map_volume_bricks(self.h, _ptr(k), _ptr(t), _ptr(c), C.c_size_t(len(k)), C.byref(n)))
        return k, t, c

    def global_mesh(self, weight_cull=8):
        """The whole map as one mesh from the map volume and the live volume (kt_get_global_mesh): (vertices, triangles [m, 3], report
        dict).  Counts first, then fetches: that runs the export twice."""
        nv = C.c_size_t(0); nt = C.c_size_t(0); rep = GlobalMeshReport()
        _check(self.lib.kt_get_global_mesh(self.h, int(weight_cull), None, C.c_size_t(0), None, C.c_size_t(0), C.byref(nv), C.byref(nt), C.byref(rep)))
        v = np.zeros(nv.value, MESH_VERTEX_DTYPE); t = np.zeros((nt.value, 3), np.uint32)
        if nv.value or nt.value:
            _check(self.lib.kt_get_global_mesh(self.h, int(weight_cull), _ptr(v), C.c_size_t(len(v)), _ptr(t), C.c_size_t(len(t)),
                                               C.byref(nv), C.byref(nt), C.byref(rep)))
        assert (nv.value, nt.value) == (len(v), len(t))
        return v, t, rep.as_dict()

    def save_global_mesh_ply(self, path, weight_cull=8):
        """The same mesh as a binary PLY in save_mesh_ply's layout (kt_save_global_mesh_ply).  Returns the report dict."""
        rep = GlobalMeshReport()
        _check(self.lib.kt_save_global_mesh_ply(self.h, os.fsencode(path), int(weight_cull), C.byref(rep)))
        return rep.as_dict()

    def live_mesh(self):
        """Mesh of the whole volume now (kt_get_live_mesh): (vertices, triangles)."""
        nv = C.c_size_t(0); nt = C.c_size_t(0)
        _check(self.lib.kt_get_live_mesh(self.h, None, C.c_size_t(0), None, C.c_size_t(0), C.byref(nv), C.byref(nt)))
        v = np.zeros(nv.value, MESH_VERTEX_DTYPE); t = np.zeros((nt.value, 3), np.uint32)
        _check(self.lib.kt_get_live_mesh(self.h, _ptr(v), C.c_size_t(len(v)), _ptr(t), C.c_size_t(len(t)), C.byref(nv), C.byref(nt)))
        assert (nv.value, nt.value) == (len(v), len(t))
        return v, t

    def save_mesh_ply(self, path):
        """Every recorded slice mesh, concatenated, as a binary PLY (kt_save_mesh_ply)."""
        _check(self.lib.kt_save_mesh_ply(self.h, os.fsencode(path)))

    def deform_map(self, corrected, points=(), node_spacing=0.8):
        """Deform every processed slice and slice mesh recorded so far to a corrected trajectory (kt_deform_map).  corrected: iterable
        of (timestamp, 4x4 pose) with timestamps from the dense pose graph; points: iterable of (time, source xyz, target xyz).
        Returns the DeformReport."""
        corrected = list(corrected); points = list(points)
        cp = (DensePose * max(len(corrected), 1))()
        for i, (ts, pose) in enumerate(corrected):
            cp[i].timestamp = int(ts); cp[i].pose[:] = [float(v) for v in np.asarray(pose, np.float32).reshape(16)]
        pp = (DeformConstraint * max(len(points), 1))()
        for i, (ts, src, dst) in enumerate(points):
            pp[i].time = int(ts); pp[i].source[:] = [float(v) for v in src]; pp[i].target[:] = [float(v) for v in dst]
        rep = DeformReport()
        _check(self.lib.kt_deform_map(self.h, cp, C.c_size_t(len(corrected)), pp, C.c_size_t(len(points)), C.c_float(node_spacing), C.byref(rep)))
        return rep

    def get_deformed_slice(self, idx):
        """Processed cloud of slice idx as deformed by the last deform_map (POINT_NORMAL_DTYPE)."""
        n = C.c_size_t(0)
        _check(self.lib.kt_get_deformed_slice(self.h, idx, None, C.c_size_t(0), C.byref(n)))
        pts = np.zeros(n.value, dtype=POINT_NORMAL_DTYPE)
        if n.value:
            _check(self.lib.kt_get_deformed_slice(self.h, idx, _ptr(pts), C.c_size_t(n.value), C.byref(n)))
        return pts

    def get_deformed_slice_mesh(self, idx):
        """Mesh vertices of slice idx as deformed by the last deform_map (MESH_VERTEX_DTYPE); the triangles are get_slice_mesh's."""
        n = C.c_size_t(0)
        _check(self.lib.kt_get_deformed_slice_mesh(self.h, idx, None, C.c_size_t(0), C.byref(n)))
        v = np.zeros(n.value, dtype=MESH_VERTEX_DTYPE)
        if n.value:
            _check(self.lib.kt_get_deformed_slice_mesh(self.h, idx, _ptr(v), C.c_size_t(n.value), C.byref(n)))
        return v

    def save_deformed_mesh_ply(self, path):
        """The deformed slice meshes of the last deform_map as one binary PLY (kt_save_deformed_mesh_ply)."""
        _check(self.lib.kt_save_deformed_mesh_ply(self.h, os.fsencode(path)))

    def map_cloud(self, which=0, dedupe=False):
        """The map as one cloud (kt_get_map_cloud): which 0 = the recorded map, 1 = the corrected map; dedupe = the reference's -nos
        voxel grid over the concatenation.  Returns (POINT_NORMAL_DTYPE array, report dict).  Counts first, then fetches: with dedupe or
        which = 1 that runs the export twice."""
        n = C.c_size_t(0); rep = MapReport()
        _check(self.lib.kt_get_map_cloud(self.h, int(which), int(dedupe), None, C.c_size_t(0), C.byref(n), C.byref(rep)))
        pts = np.zeros(n.value, dtype=POINT_NORMAL_DTYPE)
        if n.value:
            _check(self.lib.kt_get_map_cloud(self.h, int(which), int(dedupe), _ptr(pts), C.c_size_t(n.value), C.byref(n), C.byref(rep)))
        return pts[:n.value], rep.as_dict()

    def save_map_pcd(self, path, which=0, dedupe=False):
        """The same cloud as a binary .pcd (kt_save_map_pcd): the reference's <log>.pcd is which 0 with its -nos as dedupe, <log>_opt.pcd
        is which 1 without.  Returns the report dict."""
        rep = MapReport()
        _check(self.lib.kt_save_map_pcd(self.h, os.fsencode(path), int(which), int(dedupe), C.byref(rep)))
        return rep.as_dict()

    def close_loop(self, time1, time2, T, inliers1=None, inliers2=None, pose_spacing=0.0, node_spacing=0.8, isam_thresh=10.0):
        """Close a loop (kt_close_loop): T = pose of the camera at time2 in the frame of the camera at time1 (4 x 4); inliers1 / inliers2:
        [n, 3] camera-frame points seen at time1 / time2.  Returns the LoopReport (accepted, chi2, the map deformation)."""
        lc = LoopConstraint(time1=int(time1), time2=int(time2))
        lc.constraint[:] = [float(v) for v in np.asarray(T, np.float64).reshape(16)]
        a = np.ascontiguousarray(np.asarray(inliers1 if inliers1 is not None else np.zeros((0, 3)), np.float32).reshape(-1, 3))
        b = np.ascontiguousarray(np.asarray(inliers2 if inliers2 is not None else np.zeros((0, 3)), np.float32).reshape(-1, 3))
        if len(a) != len(b):
            raise ValueError("inliers1 and inliers2 must have the same length")
        lc.inliers1 = a.ctypes.data if len(a) else None; lc.inliers2 = b.ctypes.data if len(b) else None; lc.n_inliers = len(a)
        rep = LoopReport()
        _check(self.lib.kt_close_loop(self.h, C.byref(lc), C.c_float(pose_spacing), C.c_float(node_spacing), C.c_double(isam_thresh), C.byref(rep)))
        return rep

    def num_loops(self):
        return int(self.lib.kt_num_loops(self.h))

    def set_loop_detection(self, enabled=True, **kw):
        """kt_set_loop_detection with the reference's defaults, overridden by kw (LoopDetectionParams fields)."""
        p = LoopDetectionParams()
        _check(self.lib.kt_default_loop_detection(C.byref(p)))
        p.enabled = int(enabled)
        for k, v in kw.items():
            setattr(p, k, v)
        _check(self.lib.kt_set_loop_detection(self.h, C.byref(p)))

    def detect_loops(self, capacity=256):
        """kt_detect_loops: one dict per keyframe captured since the last call (PlaceResult.as_dict)."""
        out = (PlaceResult * capacity)()
        n = C.c_size_t(0)
        _check(self.lib.kt_detect_loops(self.h, out, C.c_size_t(capacity), C.byref(n)))
        return [out[i].as_dict() for i in range(n.value)]

    def num_keyframes(self):
        full = C.c_int(0)
        n = int(self.lib.kt_num_keyframes(self.h, C.byref(full)))
        return n, bool(full.value)

    def keyframe(self, idx):
        """(timestamp, dense-pose index, feature count) of keyframe idx."""
        t = C.c_uint64(0); d = C.c_int(0); f = C.c_int(0)
        _check(self.lib.kt_get_keyframe(self.h, int(idx), C.byref(t), C.byref(d), C.byref(f)))
        return int(t.value), int(d.value), int(f.value)

    def pose_graph_nodes(self):
        """[(timestamp, 4x4 world-frame pose, is_loop_pose)] of the last accepted loop's optimised pose graph (empty before one)."""
        out = []
        for i in range(int(self.lib.kt_num_pose_graph_nodes(self.h))):
            d = DensePose()
            _check(self.lib.kt_get_pose_graph_node(self.h, i, C.byref(d)))
            out.append((int(d.timestamp), np.array(d.pose, np.float32).reshape(4, 4), bool(d.is_loop_pose)))
        return out

    def slice_info(self, idx):
        """The rest of the CloudSlice record: dimension, odometry kind, camera pose at hand-over, timestamp, point count."""
        info = SliceInfo()
        _check(self.lib.kt_get_slice_info(self.h, idx, C.byref(info)))
        return info

    def trace(self, max_iters=64):
        n = C.c_int(0)
        buf = np.zeros((max_iters, 44), dtype=np.float32)
        _check(self.lib.kt_get_trace(self.h, _ptr(buf), max_iters, C.byref(n)))
        return buf[:min(n.value, max_iters)]

    def export_volume(self, tsdf=True, color=True):
        V = self.cfg.vol
        t = np.empty((V, V, V), dtype=np.int16) if tsdf else None
        c = np.empty((V, V, V, 4), dtype=np.uint8) if color else None
        _check(self.lib.kt_volume_export_reference_layout(self.h, _ptr(t), _ptr(c)))
        return t, c

    def download_map(self, which, level=0):
        rows, cols = self.cfg.rows >> level, self.cfg.cols >> level
        if which <= 3:
            out = np.empty((3, rows, cols), dtype=np.float32)
        elif which == 4:
            out = np.empty((rows, cols), dtype=np.uint16)
        elif which == 5:
            out = np.empty((rows, cols, 4), dtype=np.uint8)
        elif which == 8:
            out = np.empty((rows, cols, 4), dtype=np.float32)
        else:
            out = np.empty((rows, cols), dtype=np.float32)
        _check(self.lib.kt_download_map(self.h, which, level, _ptr(out)))
        return out

    def live_image(self):
        """getLiveImage: (shaded uint8 [rows, cols, 3], colour uint8 [rows, cols, 3], model depth uint16 [rows, cols])."""
        r, c = self.cfg.rows, self.cfg.cols
        a = np.zeros((r, c, 3), np.uint8); b = np.zeros((r, c, 3), np.uint8); d = np.zeros((r, c), np.uint16)
        _check(self.lib.kt_get_live_image(self.h, _ptr(a), _ptr(b), _ptr(d)))
        return a, b, d

    def live_tsdf(self, max_points=None):
        n = C.c_size_t(0)
        cap = max_points if max_points is not None else 3 * self.cfg.rows * self.cfg.cols
        pts = np.zeros(cap, dtype=POINT_DTYPE)
        _check(self.lib.kt_get_live_tsdf(self.h, _ptr(pts), C.c_size_t(cap), C.byref(n)))
        return pts[:min(cap, n.value)]

    def last_integrate(self):
        """(Rinv 3x3, t 3, wrap 3) of the last integration (kt_debug_last_integrate)."""
        R = np.zeros(9, np.float32); t = np.zeros(3, np.float32); w = np.zeros(3, np.int32)
        _check(self.lib.kt_debug_last_integrate(self.h, _ptr(R), _ptr(t), _ptr(w)))
        return R.reshape(3, 3), t, w

    def set_stage_timing(self, on=True):
        _check(self.lib.kt_set_stage_timing(self.h, int(on)))

    def stage_ms(self):
        ms = (C.c_float * 6)()
        _check(self.lib.kt_get_stage_ms(self.h, ms))
        return list(ms)

    def launch_count(self):
        return int(self.lib.kt_launch_count(self.h))

    def span_mark(self, which):
        _check(self.lib.kt_span_mark(self.h, int(which)))

    def span_elapsed_ms(self):
        return float(self.lib.kt_span_elapsed_ms(self.h))

    def kernel_ms(self):
        """(icp, ztable + integrate, raycast) launches alone, ms (stage timing on)"""
        a = (C.c_float * 3)()
        _check(self.lib.kt_get_kernel_ms(self.h, a))
        return [float(x) for x in a]

    def icp_kernel_ms(self):
        return float(self.lib.kt_get_icp_kernel_ms(self.h))

    # ---- z-slab sharding (one process per GPU) ----
    def mgpu_arena_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        _check(self.lib.kt_mgpu_arena_handle(self.h, buf))
        return buf.raw

    def mgpu_connect(self, handles):
        blob = b"".join(handles)
        assert len(blob) == 64 * len(handles)
        _check(self.lib.kt_mgpu_connect(self.h, C.c_char_p(blob), len(handles)))

    def mgpu_info(self):
        info = (C.c_int * 5)()
        _check(self.lib.kt_mgpu_info(self.h, info))
        return dict(world=info[0], rank=info[1], planes=info[2], block=info[3], arena_mb=info[4])

    def export_owned(self):
        """The storage planes this rank owns (the whole volume when world == 1), in local plane order: TSDF gathered out of the local
        replica, colour / weight planes as stored.  mgpu.owned_planes() gives their storage z."""
        i = self.mgpu_info(); V = self.cfg.vol
        t = np.empty((i["planes"], V, V), dtype=np.int16); c = np.empty((i["planes"], V, V, 4), dtype=np.uint8)
        _check(self.lib.kt_volume_export_reference_layout(self.h, _ptr(t), _ptr(c)))
        return t, c

    def export_tsdf_replica(self):
        """The full local TSDF replica (world > 1: every rank holds all planes)."""
        V = self.cfg.vol
        t = np.empty((V, V, V), dtype=np.int16)
        _check(self.lib.kt_mgpu_export_tsdf_replica(self.h, _ptr(t)))
        return t


class _Ops:
    """Operator API: one function per free function of the reference's cuda/internal.h:299-536.
    Arguments are torch CUDA tensors (or raw device pointers); outputs are written in place."""

    def _l(self):
        return load()

    def bilateral(self, src, dst, rows, cols):
        _check(self._l().kt_op_bilateral(_ptr(src), _ptr(dst), rows, cols, None))

    def pyrdown(self, src, dst, src_rows, src_cols):
        _check(self._l().kt_op_pyrdown(_ptr(src), _ptr(dst), src_rows, src_cols, None))

    def create_vmap(self, intr, depth, vmap, rows, cols):
        k = _f(intr); _check(self._l().kt_op_create_vmap(_ptr(k), _ptr(depth), _ptr(vmap), rows, cols, None))

    def create_nmap(self, vmap, nmap, rows, cols):
        _check(self._l().kt_op_create_nmap(_ptr(vmap), _ptr(nmap), rows, cols, None))

    def create_maps(self, intr, depth, vmap, nmap, rows, cols):
        k = _f(intr); _check(self._l().kt_op_create_maps(_ptr(k), _ptr(depth), _ptr(vmap), _ptr(nmap), rows, cols, None))

    def frontend(self, depth_raw, rgb, rows, cols, intr, angle_color, depths, vmaps, nmaps, depth_scaled=None, cw=None, rgbf=None,
                 depth_m=None, intensity=None, dIdx=None, dIdy=None):
        """The fused per-frame front end (2 launches) on caller buffers; every pyramid argument is a list of 4 CUDA tensors."""
        k = _f(intr)
        def arr(lst):
            if lst is None:
                return None
            return (C.c_void_p * 4)(*[x.data_ptr() for x in lst])
        _check(self._l().kt_op_frontend(_ptr(depth_raw), _ptr(rgb), rows, cols, _ptr(k), int(angle_color), arr(depths), arr(vmaps), arr(nmaps),
                                        _ptr(depth_scaled), _ptr(cw), _ptr(rgbf), arr(depth_m), arr(intensity), arr(dIdx), arr(dIdy), None))

    def transform_maps(self, vs, ns, R, t, vd, nd, rows, cols):
        R = _f(R); t = _f(t)
        _check(self._l().kt_op_transform_maps(_ptr(vs), _ptr(ns), _ptr(R), _ptr(t), _ptr(vd), _ptr(nd), rows, cols, None))

    def resize_vmap(self, src, dst, in_rows, in_cols):
        _check(self._l().kt_op_resize_vmap(_ptr(src), _ptr(dst), in_rows, in_cols, None))

    def resize_nmap(self, src, dst, in_rows, in_cols):
        _check(self._l().kt_op_resize_nmap(_ptr(src), _ptr(dst), in_rows, in_cols, None))

    def icp_step(self, Rcurr, tcurr, vmap_curr, nmap_curr, Rprev_inv, tprev, intr, vmap_g_prev, nmap_g_prev, rows, cols,
                 dist_thres=0.10, angle_thres=float(np.sin(np.float32(20.0) * np.float32(3.14159254) / np.float32(180.0)))):
        A = np.zeros(36, np.float32); b = np.zeros(6, np.float32); res = np.zeros(2, np.float32)
        Rc, tc, Rp, tp, k = _f(Rcurr), _f(tcurr), _f(Rprev_inv), _f(tprev), _f(intr)
        _check(self._l().kt_op_icp_step(_ptr(Rc), _ptr(tc), _ptr(vmap_curr), _ptr(nmap_curr), _ptr(Rp), _ptr(tp), _ptr(k),
                                        _ptr(vmap_g_prev), _ptr(nmap_g_prev), rows, cols, C.c_float(dist_thres), C.c_float(angle_thres),
                                        _ptr(A), _ptr(b), _ptr(res), None))
        return A.reshape(6, 6), b, res

    def integrate(self, depth_raw, rows, cols, intr, volume_size, Rinv, t, trunc, tsdf, color, vol, wrap, rgb, nmap_curr, angle_color, depth_scaled):
        k, vs, Ri, tt = _f(intr), _f(volume_size), _f(Rinv), _f(t)
        w = np.ascontiguousarray(np.asarray(wrap, dtype=np.int32))
        _check(self._l().kt_op_integrate(_ptr(depth_raw), rows, cols, _ptr(k), _ptr(vs), _ptr(Ri), _ptr(tt), C.c_float(trunc), _ptr(tsdf), _ptr(color),
                                         vol, _ptr(w), _ptr(rgb), _ptr(nmap_curr), int(angle_color), _ptr(depth_scaled), None))

    def raycast(self, intr, R, t, trunc, volume_size, tsdf, vol, vmap, nmap, rows, cols, wrap, vmap_color, color):
        k, vs, Rr, tt = _f(intr), _f(volume_size), _f(R), _f(t)
        w = np.ascontiguousarray(np.asarray(wrap, dtype=np.int32))
        _check(self._l().kt_op_raycast(_ptr(k), _ptr(Rr), _ptr(tt), C.c_float(trunc), _ptr(vs), _ptr(tsdf), vol, _ptr(vmap), _ptr(nmap), rows, cols,
                                       _ptr(w), _ptr(vmap_color), _ptr(color), None))

    def extract_slice(self, tsdf, volume_size, vol, out, capacity, wrap, color, box, subsample, real_wrap):
        vs = _f(volume_size)
        w = np.ascontiguousarray(np.asarray(wrap, dtype=np.int32)); rw = np.ascontiguousarray(np.asarray(real_wrap, dtype=np.int32))
        n = C.c_size_t(0)
        _check(self._l().kt_op_extract_slice(_ptr(tsdf), _ptr(vs), vol, _ptr(out), C.c_size_t(capacity), _ptr(w), _ptr(color),
                                             box[0], box[1], box[2], box[3], box[4], box[5], subsample, _ptr(rw), C.byref(n), None))
        return n.value

    def process_slice(self, points_dev, n, weight_cull, leaf, out_dev, capacity, k_search=20):
        """kt_op_process_slice: weight cull + voxel grid + 20-NN normals of n device-resident 32-byte points into 48-byte points."""
        cnt = C.c_size_t(0)
        _check(self._l().kt_op_process_slice(_ptr(points_dev), C.c_size_t(n), int(weight_cull), C.c_float(leaf), int(k_search), _ptr(out_dev), C.c_size_t(capacity),
                                             C.byref(cnt), None))
        return cnt.value

    def voxel_grid(self, points_dev, n, kind, leaf, out_dev, capacity):
        """kt_op_voxel_grid: pcl::VoxelGrid over n device records of kind 0 (POINT_DTYPE) / 1 (POINT_NORMAL_DTYPE) into out_dev (up to
        capacity records of the same kind).  Returns (leaves, pcl_would_skip)."""
        cnt = C.c_size_t(0); skip = C.c_int(0)
        _check(self._l().kt_op_voxel_grid(_ptr(points_dev), C.c_size_t(n), int(kind), C.c_float(leaf), _ptr(out_dev), C.c_size_t(capacity),
                                          C.byref(cnt), C.byref(skip), None))
        return cnt.value, skip.value

    def mesh_volume_into(self, tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull, verts_dev, max_verts, tris_dev, max_tris):
        """kt_op_mesh_volume into caller buffers: (status, n_verts, n_tris); status is 0 or KT_ERR_CAPACITY (nothing written)."""
        vs = _f(volume_size)
        w = np.ascontiguousarray(np.asarray(wrap, dtype=np.int32)); rw = np.ascontiguousarray(np.asarray(real_wrap, dtype=np.int32))
        nv = C.c_size_t(0); nt = C.c_size_t(0)
        st = self._l().kt_op_mesh_volume(_ptr(tsdf), _ptr(color), vol, _ptr(vs), _ptr(w), _ptr(rw), box[0], box[1], box[2], box[3], box[4], box[5],
                                         int(weight_cull), _ptr(verts_dev), C.c_size_t(max_verts), _ptr(tris_dev), C.c_size_t(max_tris),
                                         C.byref(nv), C.byref(nt), None)
        if st not in (0, KT_ERR_CAPACITY):
            _check(st)
        return st, nv.value, nt.value

    def mesh_volume(self, tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull=8):
        """Marching cubes over box (minX, maxX, minY, maxY, minZ, maxZ) of a device volume: counts first, then output buffers of
        exactly that size.  Returns host arrays (vertices MESH_VERTEX_DTYPE [n], triangles uint32 [m, 3])."""
        import torch
        st, nv, nt = self.mesh_volume_into(tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull, None, 0, None, 0)
        if st == 0:
            return np.zeros(0, MESH_VERTEX_DTYPE), np.zeros((0, 3), np.uint32)
        v = torch.empty(nv * 32, dtype=torch.uint8, device="cuda")
        t = torch.empty(max(nt, 1) * 3, dtype=torch.int32, device="cuda")
        st, nv2, nt2 = self.mesh_volume_into(tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull, v, nv, t, nt)
        _check(st)
        assert (nv2, nt2) == (nv, nt)
        return v.cpu().numpy().view(MESH_VERTEX_DTYPE).copy(), t[:3 * nt].cpu().numpy().view(np.uint32).reshape(nt, 3).copy()

    def mesh_volume_keyed_into(self, tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull, verts_dev, edges_dev, max_verts,
                               tris_dev, cells_dev, max_tris):
        """kt_op_mesh_volume_keyed into caller buffers: (status, n_verts, n_tris); status is 0 or KT_ERR_CAPACITY (nothing written)."""
        vs = _f(volume_size)
        w = np.ascontiguousarray(np.asarray(wrap, dtype=np.int32)); rw = np.ascontiguousarray(np.asarray(real_wrap, dtype=np.int32))
        nv = C.c_size_t(0); nt = C.c_size_t(0)
        st = self._l().kt_op_mesh_volume_keyed(_ptr(tsdf), _ptr(color), vol, _ptr(vs), _ptr(w), _ptr(rw), box[0], box[1], box[2], box[3], box[4],
                                               box[5], int(weight_cull), _ptr(verts_dev), _ptr(edges_dev), C.c_size_t(max_verts), _ptr(tris_dev),
                                               _ptr(cells_dev), C.c_size_t(max_tris), C.byref(nv), C.byref(nt), None)
        if st not in (0, KT_ERR_CAPACITY):
            _check(st)
        return st, nv.value, nt.value

    def mesh_volume_keyed(self, tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull=8):
        """mesh_volume plus where each vertex and triangle is: host arrays (vertices, triangles uint32 [m, 3], edges int32 [n, 4] = gx,
        gy, gz, axis, cells int32 [m, 4] = gx, gy, gz, 0), global = logical voxel + real_wrap."""
        import torch
        st, nv, nt = self.mesh_volume_keyed_into(tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull, None, None, 0, None, None, 0)
        if st == 0:
            return np.zeros(0, MESH_VERTEX_DTYPE), np.zeros((0, 3), np.uint32), np.zeros((0, 4), np.int32), np.zeros((0, 4), np.int32)
        v = torch.empty(nv * 32, dtype=torch.uint8, device="cuda"); e = torch.empty(nv * 4, dtype=torch.int32, device="cuda")
        t = torch.empty(max(nt, 1) * 3, dtype=torch.int32, device="cuda"); k = torch.empty(max(nt, 1) * 4, dtype=torch.int32, device="cuda")
        st, nv2, nt2 = self.mesh_volume_keyed_into(tsdf, color, vol, volume_size, wrap, real_wrap, box, weight_cull, v, e, nv, t, k, nt)
        _check(st)
        assert (nv2, nt2) == (nv, nt)
        return (v.cpu().numpy().view(MESH_VERTEX_DTYPE).copy(), t[:3 * nt].cpu().numpy().view(np.uint32).reshape(nt, 3).copy(),
                e.cpu().numpy().reshape(nv, 4), k[:4 * nt].cpu().numpy().reshape(nt, 4))

    def mesh_bricks_into(self, keys_dev, tsdf_dev, color_dev, n_bricks, volume_size, vol, weight_cull, verts_dev, max_verts, tris_dev, max_tris):
        """kt_op_mesh_bricks into caller buffers: (status, n_verts, n_tris); status is 0 or KT_ERR_CAPACITY (nothing written)."""
        vs = _f(volume_size)
        nv = C.c_size_t(0); nt = C.c_size_t(0)
        st = self._l().kt_op_mesh_bricks(_ptr(keys_dev), _ptr(tsdf_dev), _ptr(color_dev), C.c_size_t(n_bricks), _ptr(vs), int(vol), int(weight_cull),
                                         _ptr(verts_dev), C.c_size_t(max_verts), _ptr(tris_dev), C.c_size_t(max_tris), C.byref(nv), C.byref(nt), None)
        if st not in (0, KT_ERR_CAPACITY):
            _check(st)
        return st, nv.value, nt.value

    def mesh_bricks(self, keys, tsdf, color, volume_size, vol, weight_cull=8):
        """Marching cubes over a sorted brick set (kt_op_mesh_bricks): keys uint64 [n], tsdf int16 [n, 8, 8, 8], colour uint8 [n, 8, 8, 8, 4]
        (host arrays or CUDA tensors).  Returns host arrays (vertices MESH_VERTEX_DTYPE [n], triangles uint32 [m, 3])."""
        import torch
        dev = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()  # noqa: E731
        n = len(keys)
        dk, dt, dc = (dev(keys), dev(tsdf), dev(color)) if n else (None, None, None)
        _, nv, nt = self.mesh_bricks_into(dk, dt, dc, n, volume_size, vol, weight_cull, None, 0, None, 0)
        v = torch.empty(max(nv, 1) * 32, dtype=torch.uint8, device="cuda"); t = torch.empty(max(nt, 1) * 3, dtype=torch.int32, device="cuda")
        st, nv2, nt2 = self.mesh_bricks_into(dk, dt, dc, n, volume_size, vol, weight_cull, v, nv, t, nt)
        _check(st)
        assert (nv2, nt2) == (nv, nt)
        return v[:32 * nv].cpu().numpy().view(MESH_VERTEX_DTYPE).copy(), t[:3 * nt].cpu().numpy().view(np.uint32).reshape(nt, 3).copy()

    def weld_meshes_into(self, verts_dev, edges_dev, vert_offsets, tris_dev, cells_dev, tri_offsets, out_verts_dev, max_verts, out_tris_dev, max_tris):
        """kt_op_weld_meshes on device buffers with host offsets (n_meshes + 1 each): (status, n_verts, n_tris, report dict); status is 0
        or KT_ERR_CAPACITY (nothing written)."""
        vo = np.ascontiguousarray(np.asarray(vert_offsets, np.uint64)); to = np.ascontiguousarray(np.asarray(tri_offsets, np.uint64))
        nv = C.c_size_t(0); nt = C.c_size_t(0); rep = WeldReport()
        st = self._l().kt_op_weld_meshes(_ptr(verts_dev), _ptr(edges_dev), _ptr(vo), _ptr(tris_dev), _ptr(cells_dev), _ptr(to), len(vo) - 1,
                                         _ptr(out_verts_dev), C.c_size_t(max_verts), _ptr(out_tris_dev), C.c_size_t(max_tris), C.byref(nv), C.byref(nt),
                                         C.byref(rep), None)
        if st not in (0, KT_ERR_CAPACITY):
            _check(st)
        return st, nv.value, nt.value, rep.as_dict()

    def weld_meshes(self, meshes):
        """Weld host meshes [(vertices, triangles [m, 3], edges [n, 4], cells [m, 4])] on the device: (vertices, triangles, report dict)."""
        import torch
        cat = lambda xs, dt, w: np.ascontiguousarray(np.concatenate([np.asarray(x, dt).reshape(-1, w) for x in xs]) if xs else np.zeros((0, w), dt))  # noqa: E731
        v = np.concatenate([np.asarray(m[0]) for m in meshes]) if meshes else np.zeros(0, MESH_VERTEX_DTYPE)
        t = cat([m[1] for m in meshes], np.uint32, 3); e = cat([m[2] for m in meshes], np.int32, 4); k = cat([m[3] for m in meshes], np.int32, 4)
        vo = np.concatenate([[0], np.cumsum([len(m[0]) for m in meshes])]); to = np.concatenate([[0], np.cumsum([len(m[1]) for m in meshes])])
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda() if a.size else None  # noqa: E731
        dv, dt, de, dk = dev(v), dev(t), dev(e), dev(k)
        ov = torch.empty(max(len(v), 1) * 32, dtype=torch.uint8, device="cuda"); ot = torch.empty(max(len(t), 1) * 12, dtype=torch.uint8, device="cuda")
        st, nv, nt, rep = self.weld_meshes_into(dv, de, vo, dt, dk, to, ov, len(v), ot, len(t))
        _check(st)
        return ov[:nv * 32].cpu().numpy().view(MESH_VERTEX_DTYPE).copy(), ot[:nt * 12].cpu().numpy().view(np.uint32).reshape(nt, 3).copy(), rep

    def deform_weights(self, node_pos, node_times, points, kind, times, ids, weights):
        """kt_op_deform_weights: node_pos float32 [n, 3], node_times uint64 [n] (as int64 tensors), points (kind 0
        POINT_NORMAL records, 1 MESH_VERTEX records, 2 float32 xyz), times [N]; writes ids int32 [N, 4] and weights float64 [N, 4]."""
        _check(self._l().kt_op_deform_weights(_ptr(node_pos), _ptr(node_times), int(node_pos.shape[0]), _ptr(points), int(kind), _ptr(times),
                                              C.c_size_t(int(times.shape[0])), _ptr(ids), _ptr(weights), None))

    def deform_optimise(self, node_pos, con_src, con_dst, con_ids, con_weights, params):
        """kt_op_deform_optimise: con_src float32 [m, 3], con_dst float64 [m, 3], the sources' ids / weights; writes params float64
        [n, 12] (rotation column-major, translation).  Returns the DeformReport."""
        rep = DeformReport()
        _check(self._l().kt_op_deform_optimise(_ptr(node_pos), int(node_pos.shape[0]), _ptr(con_src), _ptr(con_dst), _ptr(con_ids),
                                               _ptr(con_weights), C.c_size_t(int(con_src.shape[0])), _ptr(params), C.byref(rep), None))
        return rep

    def deform_apply(self, node_pos, params, ids, weights, points_in, points_out, kind, n):
        """kt_op_deform_apply: n records of kind 0 (POINT_NORMAL) / 1 (MESH_VERTEX) from points_in to points_out."""
        _check(self._l().kt_op_deform_apply(_ptr(node_pos), _ptr(params), int(node_pos.shape[0]), _ptr(ids), _ptr(weights), _ptr(points_in),
                                            _ptr(points_out), int(kind), C.c_size_t(int(n)), None))

    def pgo_optimise(self, poses, factors, out):
        """kt_op_pgo_optimise: poses float64 [n, 4, 4] (device), factors PGO_FACTOR_DTYPE records as a device byte tensor; writes the
        optimised poses to out (may be poses).  Returns the PgoReport."""
        rep = PgoReport()
        n = int(poses.numel() // 16)
        _check(self._l().kt_op_pgo_optimise(_ptr(poses), n, _ptr(factors), int(factors.numel() // PGO_FACTOR_DTYPE.itemsize), _ptr(out),
                                            C.byref(rep), None))
        return rep

    def surf(self, rgb, rows, cols, max_features=1000, threshold=400.0):
        """kt_op_surf on a device RGB image: (kp float32 [n, 6] = x, y, size, angle, response, laplacian; desc float32 [n, 64])."""
        import torch
        kp = torch.empty(max_features * 6, dtype=torch.float32, device="cuda")
        desc = torch.empty(max_features * 64, dtype=torch.float32, device="cuda")
        n = C.c_int(0)
        _check(self._l().kt_op_surf(_ptr(rgb), rows, cols, C.c_float(threshold), int(max_features), _ptr(kp), _ptr(desc), C.byref(n), None))
        n = n.value
        return kp[:6 * n].cpu().numpy().reshape(n, 6), desc[:64 * n].cpu().numpy().reshape(n, 64)

    def keypoints_3d(self, kp, depth, rows, cols, intr):
        """kt_op_keypoints_3d on device keypoints kp [n, 6] and a device depth image: host float32 [n, 3], NaN rows without a point."""
        import torch
        n = int(kp.shape[0])
        xyz = torch.empty(max(n, 1) * 3, dtype=torch.float32, device="cuda")
        _check(self._l().kt_op_keypoints_3d(_ptr(kp), n, _ptr(depth), rows, cols, _ptr(_f(intr)), _ptr(xyz), None))
        return xyz[:3 * n].cpu().numpy().reshape(n, 3)

    def match_ratio(self, db, query, ratio=0.49, stride=None, seg_counts=None):
        """kt_op_match_ratio on device descriptors db [n_seg * stride, 64] (stride None: one segment of all rows), query [m, 64]; seg_counts:
        valid rows per segment (None: all).  Returns host arrays (best, d1, d2, pass, passes per segment)."""
        import torch
        n, m = int(db.shape[0]), int(query.shape[0])
        stride = n if stride is None else int(stride)
        n_seg = n // stride if stride else 0
        cnt = None if seg_counts is None else np.ascontiguousarray(np.asarray(seg_counts, np.int32))
        sp = np.zeros(max(n_seg, 1), np.int32)
        best = torch.empty(max(n, 1), dtype=torch.int32, device="cuda"); d1 = torch.empty(max(n, 1), dtype=torch.float32, device="cuda")
        d2 = torch.empty(max(n, 1), dtype=torch.float32, device="cuda"); ps = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
        _check(self._l().kt_op_match_ratio(_ptr(db), n_seg, stride, _ptr(cnt), _ptr(query), m, C.c_float(ratio), _ptr(best), _ptr(d1), _ptr(d2),
                                           _ptr(ps), _ptr(sp), None))
        return best[:n].cpu().numpy(), d1[:n].cpu().numpy(), d2[:n].cpu().numpy(), ps[:n].cpu().numpy().astype(bool), sp[:n_seg]

    def pnp_ransac(self, p_new, p_old, uv_old, intr, iterations=500, threshold_px=2.0, seed=0x4B696E74756F7573):
        """kt_op_pnp_ransac on host arrays: (R 3x3, t 3, inlier mask, n_inliers) with p_old ~ R p_new + t."""
        a, b, u = _f(p_new), _f(p_old), _f(uv_old)
        n = len(a) // 3
        pose = np.zeros(12, np.float64); inl = np.zeros(max(n, 1), np.uint8); ni = C.c_int(0)
        k = _f(intr)
        _check(self._l().kt_op_pnp_ransac(_ptr(a), _ptr(b), _ptr(u), n, _ptr(k), int(iterations), C.c_float(threshold_px), C.c_uint64(seed),
                                          _ptr(pose), _ptr(inl), C.byref(ni)))
        return pose[:9].reshape(3, 3), pose[9:].copy(), inl[:n].astype(bool), ni.value

    def cloud_fitness(self, src_depth, dst_depth, rows, cols, intr, leaf, T):
        """kt_op_cloud_fitness on device depth images (u16 mm): (fitness, n_src, n_dst) with source moved by T (3x4 or 4x4)."""
        k = _f(intr); T12 = _f(np.asarray(T, np.float64)[:3, :4])
        f = C.c_double(0); ns = C.c_size_t(0); nd = C.c_size_t(0)
        _check(self._l().kt_op_cloud_fitness(_ptr(src_depth), _ptr(dst_depth), rows, cols, _ptr(k), C.c_float(leaf), _ptr(T12), C.byref(f), C.byref(ns), C.byref(nd)))
        return f.value, ns.value, nd.value

    def clear_volume(self, axis, back, tsdf, color, vol, current, delta):
        _check(self._l().kt_op_clear_volume(axis, back, _ptr(tsdf), _ptr(color), vol, current, delta, None))

    def init_volume(self, tsdf, color, vol):
        _check(self._l().kt_op_init_volume(_ptr(tsdf), _ptr(color), vol, None))

    def short_depth_to_metres(self, src, dst, rows, cols, cut_off):
        _check(self._l().kt_op_short_depth_to_metres(_ptr(src), _ptr(dst), rows, cols, cut_off, None))

    def pyrdown_gauss_f(self, src, dst, src_rows, src_cols):
        _check(self._l().kt_op_pyrdown_gauss_f(_ptr(src), _ptr(dst), src_rows, src_cols, None))

    def bgr_to_intensity(self, rgb, dst, rows, cols):
        _check(self._l().kt_op_bgr_to_intensity(_ptr(rgb), _ptr(dst), rows, cols, None))

    def pyrdown_uchar_gauss(self, src, dst, src_rows, src_cols):
        _check(self._l().kt_op_pyrdown_uchar_gauss(_ptr(src), _ptr(dst), src_rows, src_cols, None))

    def derivative_images(self, src, dx, dy, rows, cols):
        _check(self._l().kt_op_derivative_images(_ptr(src), _ptr(dx), _ptr(dy), rows, cols, None))

    def project_to_point_cloud(self, depth, cloud, rows, cols, intr_d, level):
        k = np.ascontiguousarray(np.asarray(intr_d, dtype=np.float64))
        _check(self._l().kt_op_project_to_point_cloud(_ptr(depth), _ptr(cloud), rows, cols, _ptr(k), level, None))

    def rgb_residual(self, min_scale, dIdx, dIdy, last_depth, next_depth, last_image, next_image, corres, rows, cols, max_depth_delta, kt, krkinv):
        ktf, kk = _f(kt), _f(krkinv)
        sigma = C.c_int(0); count = C.c_int(0)
        _check(self._l().kt_op_rgb_residual(C.c_float(min_scale), _ptr(dIdx), _ptr(dIdy), _ptr(last_depth), _ptr(next_depth), _ptr(last_image), _ptr(next_image),
                                            _ptr(corres), rows, cols, C.c_float(max_depth_delta), _ptr(ktf), _ptr(kk), C.byref(sigma), C.byref(count), None))
        return sigma.value, count.value

    def generate_image(self, vmap, nmap, vmap_color, light_pos, n_lights, dst, dst_color, rows, cols):
        lp = _f(light_pos)
        _check(self._l().kt_op_generate_image(_ptr(vmap), _ptr(nmap), _ptr(vmap_color), _ptr(lp), n_lights, _ptr(dst), _ptr(dst_color), rows, cols, None))

    def generate_depth(self, Rinv, t, vmap, nmap, dst, rows, cols, max_depth=6.0):
        Ri, tt = _f(Rinv), _f(t)
        _check(self._l().kt_op_generate_depth(_ptr(Ri), _ptr(tt), _ptr(vmap), _ptr(nmap), _ptr(dst), rows, cols, C.c_float(max_depth), None))

    def rgb_step(self, corres, sigma, cloud, fx, fy, dIdx, dIdy, sobel_scale, rows, cols):
        A = np.zeros(36, np.float32); b = np.zeros(6, np.float32)
        _check(self._l().kt_op_rgb_step(_ptr(corres), C.c_float(sigma), _ptr(cloud), C.c_float(fx), C.c_float(fy), _ptr(dIdx), _ptr(dIdy),
                                        C.c_float(sobel_scale), rows, cols, _ptr(A), _ptr(b), None))
        return A.reshape(6, 6), b


ops = _Ops()
