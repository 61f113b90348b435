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


class PgoReport(C.Structure):
    """kt_pgo_report of kt_op_pgo_optimise."""
    _fields_ = [("nodes", C.c_int), ("factors", C.c_int), ("loops", C.c_int), ("iterations", C.c_int),
                ("chi2_initial", C.c_double), ("chi2_final", C.c_double), ("solver_failed", C.c_int), ("step_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# kt_pgo_factor (56 bytes): i = -1 for the prior on node j
PGO_FACTOR_DTYPE = np.dtype([("i", "<i4"), ("j", "<i4"), ("z", "<f8", (6,))])
assert PGO_FACTOR_DTYPE.itemsize == 56


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
