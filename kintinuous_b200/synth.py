"""Deterministic synthetic RGB-D stream (SURVEY.md section 8d, BASELINE.md section 4).

The reference ships no data (its sample log is a download, README.md:166-170), so the workload is an
analytic scene rendered exactly: the interior of an axis-aligned 5 x 3 x 5 m room centred on the
first camera, a sphere (r = 0.5 m) and a 1 m cube standing on the floor, textured with a smooth
procedural pattern plus a 7.85 cm checker (edges strong enough for the photometric odometry's gradient test).

Camera: fx = fy = 528.01442863461716, cx = 320, cy = 267 (reference default,
MainController.cpp:222-227), scaled with the resolution.  Trajectory of frame k (camera -> world):
translation (0.010 k, 0.002 sin(k / 10), 0.004 k) m, rotation 0.2 deg * k about +y.  Depth is the
z of the hit point in the camera frame, uint16 millimetres (0 = no return beyond 6 m); colour is
uint8 RGB in the reference's PixelRGB order.  Optional Kinect-like axial noise uses
numpy.random.default_rng(SEED + k).  Pure numpy: host-side test / bench input only.
"""
from __future__ import annotations

import numpy as np

SEED = 20260922
FX = FY = 528.01442863461716
CX, CY = 320.0, 267.0

ROOM_HALF = np.array([2.5, 1.5, 2.5])
SPHERE_C = np.array([-0.6, 0.3, 1.6])
SPHERE_R = 0.5
CUBE_LO = np.array([0.4, 0.5, 1.4])
CUBE_HI = np.array([1.4, 1.5, 2.4])


def intrinsics(cols: int = 640, rows: int = 480):
    sx, sy = cols / 640.0, rows / 480.0
    return FX * sx, FY * sy, CX * sx, CY * sy


def pose(k: int):
    """Ground-truth camera-to-world pose of frame k (world = first camera frame)."""
    a = np.deg2rad(0.2 * k)
    R = np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]])
    t = np.array([0.010 * k, 0.002 * np.sin(k / 10.0), 0.004 * k])
    return R, t


def _texture(p):
    out = np.empty(p.shape[:-1] + (3,), dtype=np.float64)
    # 7.85 cm checker cells give the photometric odometry edges above its gradient threshold
    # (RGBDOdometry.cpp:109-113: |grad|^2 >= (12*8)^2 at level 0); the smooth term keeps every pixel distinct.
    sq = np.sign(np.sin(40.0 * p[..., 0] + 0.3)) * np.sign(np.sin(40.0 * p[..., 1] + 0.7)) * np.sign(np.sin(40.0 * p[..., 2] + 1.1))
    for c, ph in enumerate((0.0, 2.1, 4.2)):
        out[..., c] = 128.0 + 55.0 * np.sin(7.0 * p[..., 0] + ph) * np.sin(5.0 * p[..., 1] + 0.5 * ph) * np.sin(6.0 * p[..., 2] - ph) + 60.0 * sq
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def cell_texture(p, cell: float = 0.05):
    """Opt-in aperiodic texture (render_at's `texture`): cells of the world grid `cell` metres wide, each a grey level drawn from a hash of
    the cell's integer coordinates.  The default texture's checker repeats every 15.7 cm, so most SURF features there have look-alikes."""
    i = np.floor(p / cell).astype(np.int64)
    h = (((i[..., 0] * 73856093) ^ (i[..., 1] * 19349663) ^ (i[..., 2] * 83492791)) * 0x45D9F3B) & 0xFFFFFFFF
    return np.repeat(np.rint((((h >> 16) ^ h) & 0xFFFF) * (255.0 / 65535.0))[..., None], 3, -1).astype(np.uint8)


def render(k: int, cols: int = 640, rows: int = 480, noise: bool = False):
    """Returns (depth uint16 [rows, cols] in mm, rgb uint8 [rows, cols, 3]) of frame k of the default trajectory."""
    R, t = pose(k)
    return render_at(R, t, cols, rows, noise, noise_seed=k)


def render_at(R, t, cols: int = 640, rows: int = 480, noise: bool = False, noise_seed: int = 0, texture=None):
    """The scene seen by a camera at any pose (R, t camera -> world); the axial noise draws from default_rng(SEED + noise_seed).
    texture: optional replacement of the default texture function (world points [..., 3] -> uint8 RGB [..., 3])."""
    fx, fy, cx, cy = intrinsics(cols, rows)
    R = np.asarray(R, np.float64); t = np.asarray(t, np.float64)
    u, v = np.meshgrid(np.arange(cols, dtype=np.float64), np.arange(rows, dtype=np.float64))
    dc = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)], axis=-1)       # camera-frame ray, z = 1
    d = dc @ R.T                                                                  # world direction (not normalised)
    o = t
    with np.errstate(divide="ignore", invalid="ignore"):
        # room, seen from inside: first exit of the slab
        tt = np.where(d > 0, (ROOM_HALF - o) / d, (-ROOM_HALF - o) / d)
        t_hit = np.min(np.where(d == 0, np.inf, tt), axis=-1)
        # sphere
        oc = o - SPHERE_C
        a = np.sum(d * d, axis=-1)
        b = 2.0 * (d @ oc)
        c = float(oc @ oc) - SPHERE_R ** 2
        disc = b * b - 4 * a * c
        ts = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
        ts = np.where(ts > 1e-6, ts, np.inf)
        t_hit = np.minimum(t_hit, ts)
        # cube (from outside): slab test
        t1 = (CUBE_LO - o) / d
        t2 = (CUBE_HI - o) / d
        tn = np.max(np.minimum(t1, t2), axis=-1)
        tf = np.min(np.maximum(t1, t2), axis=-1)
        tcube = np.where((tn < tf) & (tn > 1e-6), tn, np.inf)
        t_hit = np.minimum(t_hit, tcube)
    # with a z = 1 camera ray, the ray parameter IS the camera-frame depth
    z = t_hit
    p = o + d * t_hit[..., None]
    rgb = (texture or _texture)(p)
    if noise:
        rng = np.random.default_rng(SEED + noise_seed)
        sigma = 0.0012 + 0.0019 * (z - 0.4) ** 2
        z = z + rng.standard_normal(z.shape) * sigma
    mm = np.rint(1000.0 * z)
    depth = np.where((z > 0) & (z <= 6.0) & np.isfinite(z), mm, 0).astype(np.uint16)
    return depth, rgb


def sequence(n: int, cols: int = 640, rows: int = 480, noise: bool = False, start: int = 0):
    for k in range(start, start + n):
        d, c = render(k, cols, rows, noise)
        yield k, d, c
