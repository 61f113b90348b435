"""TEST INFRASTRUCTURE ONLY (oracle/): ctypes bindings of the two oracles.

  * RefCuda  -- oracle/_ref/libkt_ref_<VOL>.so: the reference's OWN CUDA operators (compiled by
                oracle/build_ref.sh from the reference checkout) behind oracle/ref_harness.cu.  Needs a GPU.
  * CpuOracle -- oracle/libkt_oracle_cpu.so: the CPU restatement (oracle/kt_oracle_cpu.cpp).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
The product (kintinuous_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


class TrackerConfig(C.Structure):
    """kto::TrackerConfig (oracle/kt_host_logic.hpp)."""
    _fields_ = [("rows", C.c_int), ("cols", C.c_int), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("vol", C.c_int), ("volume_size", C.c_float), ("odometry", C.c_int), ("fast_odometry", C.c_int),
                ("voxel_shift", C.c_int), ("overlap", C.c_int), ("angle_color", C.c_int), ("parked", C.c_int), ("cloud_capacity", C.c_int)]

    @staticmethod
    def from_kt(cfg):
        cap = cfg.cloud_capacity if cfg.cloud_capacity > 0 else 3 * cfg.rows * cfg.cols
        return TrackerConfig(cfg.rows, cfg.cols, cfg.fx, cfg.fy, cfg.cx, cfg.cy, cfg.vol, cfg.volume_size, cfg.odometry, cfg.fast_odometry,
                             cfg.voxel_shift, cfg.overlap, cfg.angle_color, cfg.parked, cap)


POINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("_p0", "<f4"),
                        ("b", "u1"), ("g", "u1"), ("r", "u1"), ("a", "u1"), ("_p1", "u1", (12,))])


def _ptr(a):
    if a is None:
        return C.c_void_p(0)
    if isinstance(a, int):
        return C.c_void_p(a)
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(a.data_ptr())


def _f(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(-1))


def _i(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.int32).reshape(-1))


class _TrackerBase:
    prefix = ""

    def __init__(self, lib, cfg: TrackerConfig):
        self.lib = lib
        self.cfg = cfg
        self._fn("create").restype = C.c_void_p
        self._fn("get_slice").restype = C.c_size_t
        self._fn("trunc_dist").restype = C.c_float
        self.h = C.c_void_p(self._fn("create")(C.byref(cfg)))

    def _fn(self, name):
        return getattr(self.lib, self.prefix + name)

    def close(self):
        if self.h:
            self._fn("destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process(self, depth: np.ndarray, rgb: np.ndarray, utime=0):
        self._fn("process")(self.h, _ptr(depth), _ptr(rgb), C.c_uint64(utime))

    def finalise(self):
        self._fn("finalise")(self.h)

    def pose(self):
        R = np.zeros(9, np.float32); t = np.zeros(3, np.float32); g = np.zeros(3, np.float32); w = np.zeros(3, np.int32)
        self._fn("get_pose")(self.h, _ptr(R), _ptr(t), _ptr(g), _ptr(w))
        return R.reshape(3, 3), t, g, w

    @property
    def trunc_dist(self):
        return float(self._fn("trunc_dist")(self.h))

    def export_volume(self, tsdf=True, color=True):
        V = self.cfg.vol
        t = np.empty((V, V, V), np.int16) if tsdf else None
        c = np.empty((V, V, V, 4), np.uint8) if color else None
        self._fn("download_volume")(self.h, _ptr(t), _ptr(c))
        return t, c

    def download_map(self, which, level=0):
        rows, cols = self.cfg.rows >> level, self.cfg.cols >> level
        out = np.empty((3, rows, cols), np.float32) if which <= 3 else (np.empty((rows, cols), np.uint16) if which == 4 else np.empty((rows, cols, 4), np.uint8))
        self._fn("download_map")(self.h, which, level, _ptr(out))
        return out

    def trace(self, max_iters=64):
        buf = np.zeros((max_iters, 44), np.float32)
        n = self._fn("trace")(self.h, _ptr(buf), max_iters)
        return buf[:min(n, max_iters)]

    def num_slices(self):
        return int(self._fn("num_slices")(self.h))

    def get_slice(self, idx):
        dim = C.c_int(0); cam = (C.c_float * 3)()
        n = self._fn("get_slice")(self.h, idx, None, C.c_size_t(0), C.byref(dim), cam)
        pts = np.zeros(n, dtype=POINT_DTYPE)
        if n:
            self._fn("get_slice")(self.h, idx, _ptr(pts), C.c_size_t(n), C.byref(dim), cam)
        return pts, dim.value, np.array(cam, np.float32)


class RefCuda:
    """The reference's own CUDA operators (GPU required)."""

    def __init__(self, vol: int):
        p = os.path.join(_HERE, "_ref", f"libkt_ref_{vol}.so")
        if not os.path.exists(p):
            raise FileNotFoundError(f"{p}: run oracle/build_ref.sh {vol} where the reference checkout exists")
        self.lib = C.CDLL(p)
        self.lib.ktref_extract.restype = C.c_size_t
        self.vol = self.lib.ktref_vol()
        assert self.vol == vol

    @staticmethod
    def available(vol: int) -> bool:
        return os.path.exists(os.path.join(_HERE, "_ref", f"libkt_ref_{vol}.so"))

    def tracker(self, cfg: TrackerConfig):
        t = _TrackerBase.__new__(_TrackerBase)
        t.prefix = "ktref_tracker_"
        _TrackerBase.__init__(t, self.lib, cfg)
        return t

    # ---- operators (device pointers / torch CUDA tensors) ----
    def bilateral(self, src, dst, rows, cols): self.lib.ktref_bilateral(_ptr(src), _ptr(dst), rows, cols)
    def pyrdown(self, src, dst, sr, sc): self.lib.ktref_pyrdown(_ptr(src), _ptr(dst), sr, sc)
    def vmap(self, depth, vmap, rows, cols, intr): k = _f(intr); self.lib.ktref_vmap(_ptr(depth), _ptr(vmap), rows, cols, _ptr(k))
    def nmap(self, vmap, nmap, rows, cols): self.lib.ktref_nmap(_ptr(vmap), _ptr(nmap), rows, cols)

    def transform_maps(self, vs, ns, R, t, vd, nd, rows, cols):
        R = _f(R); t = _f(t); self.lib.ktref_transform_maps(_ptr(vs), _ptr(ns), _ptr(R), _ptr(t), _ptr(vd), _ptr(nd), rows, cols)

    def resize_vmap(self, a, b, r, c): self.lib.ktref_resize_vmap(_ptr(a), _ptr(b), r, c)
    def resize_nmap(self, a, b, r, c): self.lib.ktref_resize_nmap(_ptr(a), _ptr(b), r, c)

    def icp_step(self, Rcurr, tcurr, vmap_curr, nmap_curr, Rprev_inv, tprev, intr, vmap_g_prev, nmap_g_prev, rows, cols,
                 dist_thres=0.10, angle_thres=float(np.sin(np.float32(20.0) * np.float32(3.14159254) / np.float32(180.0)))):
        A = np.zeros(36, np.float32); b = np.zeros(6, np.float32); res = np.zeros(2, np.float32)
        Rc, tc, Rp, tp, k = _f(Rcurr), _f(tcurr), _f(Rprev_inv), _f(tprev), _f(intr)
        self.lib.ktref_icp_step(_ptr(Rc), _ptr(tc), _ptr(vmap_curr), _ptr(nmap_curr), _ptr(Rp), _ptr(tp), _ptr(k), _ptr(vmap_g_prev), _ptr(nmap_g_prev),
                                rows, cols, C.c_float(dist_thres), C.c_float(angle_thres), _ptr(A), _ptr(b), _ptr(res))
        return A.reshape(6, 6), b, res

    def integrate(self, depth_raw, rows, cols, intr, volume_size, Rinv, t, trunc, tsdf, color, wrap, rgb, nmap_curr, angle_color, depth_scaled):
        k, vs, Ri, tt, w = _f(intr), _f(volume_size), _f(Rinv), _f(t), _i(wrap)
        self.lib.ktref_integrate(_ptr(depth_raw), rows, cols, _ptr(k), _ptr(vs), _ptr(Ri), _ptr(tt), C.c_float(trunc), _ptr(tsdf), _ptr(color), _ptr(w),
                                 _ptr(rgb), _ptr(nmap_curr), int(angle_color), _ptr(depth_scaled))

    def raycast(self, intr, R, t, trunc, volume_size, tsdf, vmap, nmap, rows, cols, wrap, vmap_color, color):
        k, vs, Rr, tt, w = _f(intr), _f(volume_size), _f(R), _f(t), _i(wrap)
        self.lib.ktref_raycast(_ptr(k), _ptr(Rr), _ptr(tt), C.c_float(trunc), _ptr(vs), _ptr(tsdf), _ptr(vmap), _ptr(nmap), rows, cols, _ptr(w), _ptr(vmap_color), _ptr(color))

    def extract(self, tsdf, volume_size, out, capacity, wrap, color, box, subsample, real_wrap):
        vs, w, rw = _f(volume_size), _i(wrap), _i(real_wrap)
        return int(self.lib.ktref_extract(_ptr(tsdf), _ptr(vs), _ptr(out), C.c_size_t(capacity), _ptr(w), _ptr(color),
                                          box[0], box[1], box[2], box[3], box[4], box[5], subsample, _ptr(rw)))

    def generate_image(self, vmap, nmap, vmap_color, light_pos, n_lights, dst, dst_color, rows, cols):
        lp = _f(light_pos); self.lib.ktref_generate_image(_ptr(vmap), _ptr(nmap), _ptr(vmap_color), _ptr(lp), n_lights, _ptr(dst), _ptr(dst_color), rows, cols)

    def generate_depth(self, Rinv, t, vmap, nmap, dst, rows, cols, max_depth=6.0):
        Ri, tt = _f(Rinv), _f(t); self.lib.ktref_generate_depth(_ptr(Ri), _ptr(tt), _ptr(vmap), _ptr(nmap), _ptr(dst), rows, cols, C.c_float(max_depth))

    def clear(self, axis, back, tsdf, color, current, delta): self.lib.ktref_clear(axis, back, _ptr(tsdf), _ptr(color), current, delta)
    def init_volume(self, tsdf, color): self.lib.ktref_init_volume(_ptr(tsdf), _ptr(color))
    def short_depth_to_metres(self, s, d, rows, cols, cut): self.lib.ktref_short_depth_to_metres(_ptr(s), _ptr(d), rows, cols, cut)
    def pyrdown_gauss_f(self, s, d, sr, sc): self.lib.ktref_pyrdown_gauss_f(_ptr(s), _ptr(d), sr, sc)
    def bgr_to_intensity(self, s, d, rows, cols): self.lib.ktref_bgr_to_intensity(_ptr(s), _ptr(d), rows, cols)
    def pyrdown_uchar_gauss(self, s, d, sr, sc): self.lib.ktref_pyrdown_uchar_gauss(_ptr(s), _ptr(d), sr, sc)
    def derivative_images(self, s, dx, dy, rows, cols): self.lib.ktref_derivative_images(_ptr(s), _ptr(dx), _ptr(dy), rows, cols)

    def project_to_point_cloud(self, depth, cloud, rows, cols, intr_d, level):
        k = np.ascontiguousarray(np.asarray(intr_d, np.float64)); self.lib.ktref_project_to_point_cloud(_ptr(depth), _ptr(cloud), rows, cols, _ptr(k), level)

    def rgb_residual(self, min_scale, dIdx, dIdy, last_depth, next_depth, last_image, next_image, corres, rows, cols, max_depth_delta, kt, krkinv):
        ktf, kk = _f(kt), _f(krkinv); sigma = C.c_int(0); count = C.c_int(0)
        self.lib.ktref_rgb_residual(C.c_float(min_scale), _ptr(dIdx), _ptr(dIdy), _ptr(last_depth), _ptr(next_depth), _ptr(last_image), _ptr(next_image),
                                    _ptr(corres), rows, cols, C.c_float(max_depth_delta), _ptr(ktf), _ptr(kk), C.byref(sigma), C.byref(count))
        return sigma.value, count.value

    def rgb_step(self, corres, sigma, cloud, fx, fy, dIdx, dIdy, sobel_scale, rows, cols):
        A = np.zeros(36, np.float32); b = np.zeros(6, np.float32)
        self.lib.ktref_rgb_step(_ptr(corres), C.c_float(sigma), _ptr(cloud), C.c_float(fx), C.c_float(fy), _ptr(dIdx), _ptr(dIdy), C.c_float(sobel_scale), rows, cols, _ptr(A), _ptr(b))
        return A.reshape(6, 6), b


class CpuOracle:
    """CPU restatement (oracle/kt_oracle_cpu.cpp); all pointers are host numpy arrays."""

    def __init__(self):
        p = os.path.join(_HERE, "libkt_oracle_cpu.so")
        if not os.path.exists(p):
            raise FileNotFoundError(f"{p}: run make -C oracle")
        self.lib = C.CDLL(p)

    @staticmethod
    def available() -> bool:
        return os.path.exists(os.path.join(_HERE, "libkt_oracle_cpu.so"))

    def tracker(self, cfg: TrackerConfig):
        t = _TrackerBase.__new__(_TrackerBase)
        t.prefix = "ktoracle_tracker_"
        _TrackerBase.__init__(t, self.lib, cfg)
        return t


POINT_NORMAL_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("_p0", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"), ("_p1", "<f4"),
                               ("b", "u1"), ("g", "u1"), ("r", "u1"), ("a", "u1"), ("curvature", "<f4"), ("_p2", "<f4", (2,))])


class SliceOracle:
    """CPU restatement of CloudSliceProcessor's per-slice post-processing (oracle/kt_slice_oracle.cpp: weight cull, pcl::VoxelGrid,
    pcl::NormalEstimation of PCL 1.7.2).  Host numpy arrays of POINT_DTYPE in, POINT_NORMAL_DTYPE out."""

    def __init__(self):
        p = os.path.join(_HERE, "libkt_slice_oracle.so")
        if not os.path.exists(p):
            raise FileNotFoundError(f"{p}: run make -C oracle")
        self.lib = C.CDLL(p)
        for f in ("ktslice_weight_cull", "ktslice_voxel_grid", "ktslice_process"):
            getattr(self.lib, f).restype = C.c_size_t

    def weight_cull(self, pts, weight_cull):
        out = np.zeros(len(pts), POINT_DTYPE)
        n = self.lib.ktslice_weight_cull(_ptr(pts), C.c_size_t(len(pts)), int(weight_cull), _ptr(out))
        return out[:n]

    def voxel_grid(self, pts, leaf):
        out = np.zeros(len(pts), POINT_DTYPE); mb = np.zeros(3, np.int32); db = np.zeros(3, np.int32)
        n = self.lib.ktslice_voxel_grid(_ptr(pts), C.c_size_t(len(pts)), C.c_float(leaf), _ptr(out), C.c_size_t(len(pts)), _ptr(mb), _ptr(db))
        return out[:n], mb, db

    def normals(self, pts, k, cell):
        out = np.zeros(len(pts), POINT_NORMAL_DTYPE)
        self.lib.ktslice_normals(_ptr(pts), C.c_size_t(len(pts)), int(k), C.c_float(cell), _ptr(out))
        return out

    def process(self, pts, weight_cull, leaf, k=20):
        out = np.zeros(max(1, len(pts)), POINT_NORMAL_DTYPE)
        n = self.lib.ktslice_process(_ptr(pts), C.c_size_t(len(pts)), int(weight_cull), C.c_float(leaf), int(k), _ptr(out), C.c_size_t(len(out)))
        return out[:n]

    def eigen33(self, cov):
        c = np.ascontiguousarray(np.asarray(cov, np.float32).reshape(9)); ev = C.c_float(0); vec = np.zeros(3, np.float32)
        self.lib.ktslice_eigen33(_ptr(c), C.byref(ev), _ptr(vec))
        return ev.value, vec
