"""The volume operators over a fixed table of views (tests/test_gpu_volume_views.py, tools/make_golden.py).

Each view is a camera pose in the volume frame and the voxel wrap it is integrated with.  run_view() integrates two frames (the view, then
a perturbed pose), ray casts from both poses, extracts slabs touching both ends of each axis and clears runs of planes along each axis, on
whatever operators it is given: the reference's (make_golden records the outputs) or the product's (the test requires the same outputs,
bit for bit).  The table reaches what the tracker's forward trajectory never does: viewing axes along -z, +-x, +-y (Rinv.r2.z exactly
-1, 0 and 1), rays that enter the cube from outside or leave it through a side face, a camera on a face and one looking away from the
cube, and volume sides that are not powers of two (96, 384) or not even multiples of 32 (200), with the storage seams placed through
the observed surface."""
import numpy as np

import digest

VOLS = (96, 200, 256, 384)
SIZE = 6.0
ROWS, COLS = 120, 160
ANISO = (6.0, 4.5, 3.3)                   # one anisotropic cube at 256^3, three views
ANISO_VIEWS = ("pz", "oblique_up", "px")
CAP = 2_000_000                           # extraction capacity (points); the reference writes past its buffer, so it must never be reached


def _rot(axis, ang):
    a = np.asarray(axis, np.float64); a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _look(d, up=(0.0, 1.0, 0.0)):
    """camera -> volume rotation whose camera z looks along d (camera y as close to `up` as possible)"""
    z = np.asarray(d, np.float64); z = z / np.linalg.norm(z)
    x = np.cross(np.asarray(up, np.float64), z); x = x / np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], 1)


# exact sign / permutation matrices (columns: camera x, y, z in the volume frame), so that r2.z of R^T is exactly 1, -1 or 0
_AXIS = {
    "pz": np.eye(3),
    "mz": np.diag([-1.0, 1.0, -1.0]),
    "px": np.array([[0.0, 0, 1], [0, 1, 0], [-1, 0, 0]]),
    "mx": np.array([[0.0, 0, -1], [0, 1, 0], [1, 0, 0]]),
    "py": np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]]),
    "my": np.array([[1.0, 0, 0], [0, 0, -1], [0, 1, 0]]),
}
AXIS_VIEWS = tuple(_AXIS)


def views(V, vs=(SIZE, SIZE, SIZE)):
    """[(name, R camera->volume float32, t float32, wrap)] for a V^3 volume of size vs.  Wraps are non-negative (as the tracker passes
    them); `seam` puts each axis' storage seam (logical voxel V - wrap) through the room's walls, which span the middle of every axis."""
    c = np.asarray(vs, np.float64) / 2
    seam = (V - (11 * V) // 20, V - (9 * V) // 20, V - (9 * V) // 10)
    big = tuple(s + k * V for s, k in zip(seam, (1, 2, 3)))             # >= V on every axis
    mult = (V, 2 * V, V)                                                # whole volume lengths: storage = logical
    t = []
    for i, name in enumerate(AXIS_VIEWS):
        t.append((name, _AXIS[name], c, ((0, 0, 0), seam, big, mult, seam, big)[i]))
    R_up = _rot((0.3, 0.8, 0.5), 0.7)                                   # every entry non-zero, r2.z > 0
    R_dn = _rot((0.7, 0.4, 0.2), 2.3)                                   # every entry non-zero, r2.z < 0
    t.append(("oblique_up", R_up, c + np.array([0.1, -0.2, 0.15]), big))
    t.append(("oblique_down", R_dn, c + np.array([-0.15, 0.1, 0.2]), seam))
    t.append(("corner", _look(c - 0.3), np.array([0.3, 0.3, 0.3]), seam))     # near the (0, 0, 0) corner, looking at the centre
    t.append(("on_face", np.eye(3), np.array([0.0, c[1], c[2] - 1.0]), big))    # t.x = 0, looking along the x = 0 face
    t.append(("outside_z0", _rot((1, 0, 0), 0.05), np.array([c[0], c[1], -1.5]), seam))           # in through the z = 0 face
    t.append(("outside_xmax", _AXIS["mx"] @ _rot((0, 1, 0), 0.1), np.array([2 * c[0] + 1.5, c[1], c[2]]), big))  # in through x = max
    t.append(("look_away", _AXIS["mz"], np.array([c[0], c[1], -1.5]), seam))   # outside, facing away: nothing touched, nothing hit
    t.append(("face_xmax", _AXIS["mx"], np.array([2 * c[0] + 1.5, c[1], c[2]]), seam))   # in through x = max onto a wall on that face
    for name, R, _, _ in t:
        assert np.linalg.det(R) > 0.999 and np.allclose(R.T @ R, np.eye(3)), name
    assert (_rot((0.3, 0.8, 0.5), 0.7) != 0).all() and _rot((0.3, 0.8, 0.5), 0.7)[2, 2] > 0
    assert (_rot((0.7, 0.4, 0.2), 2.3) != 0).all() and _rot((0.7, 0.4, 0.2), 2.3)[2, 2] < 0
    return [(n, np.asarray(R, np.float32), np.asarray(tt, np.float32), tuple(int(w) for w in wr)) for n, R, tt, wr in t]


def table():
    """(V, volume_size, view names) of every case"""
    out = [(V, (SIZE,) * 3, [v[0] for v in views(V)]) for V in VOLS]
    out.append((256, ANISO, list(ANISO_VIEWS)))
    return out


def case_key(V, vs):
    return f"{V}" if tuple(vs) == (SIZE,) * 3 else f"{V}_aniso"


def perturbed(R, t):
    R2 = (R.astype(np.float64) @ _rot((0.3, -0.5, 0.8), 0.03)).astype(np.float32)
    return R2, (t + np.array([0.04, -0.03, 0.05], np.float32)).astype(np.float32)


def _frame(R, t, vs, cols, rows, tw=None):
    """depth / colour the scene shows from (R, t): rendered from the nearest pose inside the room, or from tw (the integration pose may be
    outside the room; the operators do not need the two to agree)"""
    from kintinuous_b200 import synth
    if tw is None:
        tw = np.clip(t.astype(np.float64) - np.asarray(vs, np.float64) / 2, -synth.ROOM_HALF + 0.2, synth.ROOM_HALF - 0.2)
    return synth.render_at(R.astype(np.float64), tw, cols, rows)


def _render_t(name, V, vs):
    """face_xmax: rendered 1.5 m + one voxel in front of the room's x = -2.5 m wall, so that integrated from 1.5 m outside the x = max
    face the wall lies between the centres of the last two voxels: the march's first voxel (the start clamp) and the next have opposite
    signs.  Every other view: None."""
    if name != "face_xmax":
        return None
    return np.array([-1.0 + vs[0] / V, 0.0, 0.0])


def trunc_of(V, vs):
    voxel = np.float32(max(vs)) / np.float32(V)
    return float(max(np.float32(0.06), np.float32(2.1) * voxel))


def slabs(V):
    """boxes touching both ends of each axis (the z one at the top reaches maxZ = V: its +z neighbour is plane 0, quirk Q12)"""
    w = max(8, V // 8)
    return {"x_lo": (0, w, 0, V, 0, V), "x_hi": (V - w, V, 0, V, 0, V), "y_lo": (0, V, 0, w, 0, V), "y_hi": (0, V, V - w, V, 0, V),
            "z_lo": (0, V, 0, V, 0, w), "z_hi": (0, V, 0, V, V - w, V)}


def clear_runs(V):
    """(axis, back, current, delta) runs: forward and back along every axis, crossing the end (and the start) of storage, and an x run
    of 16 planes (the reach quirk Q13 drops its last plane).  The reference's clearVolumeX launches 16-row blocks without a row check
    (tsdf_volume.cu:86-116), so it only stays inside the volume when V % 16 == 0: x runs are only recorded there.  Its clearVolumeXBack
    sizes the launch as n + 16 - n % 16 for n < 0 (tsdf_volume.cu:170-203): an empty or negative grid for 16 < |n| that is not a
    multiple of 16, which the tracker's shift of 14 never asks for, so the long back run is not made along x."""
    runs = []
    for axis in range(3):
        if axis == 0 and V % 16:
            continue
        runs += [(axis, 0, 2 * V - 5, 2 * V + 9), (axis, 1, 3, -11), (axis, 0, 7, 40)]
        if axis:
            runs.append((axis, 1, V + 20, V - 17))
    if V % 16 == 0:
        runs += [(0, 0, V - 8, V + 8), (0, 1, 5, -27)]
    return runs


def sample(n, k, seed):
    return np.sort(np.random.default_rng(seed).choice(n, size=min(k, n), replace=False))


def run_view(ops, torch, V, vs, name, R, t, wrap):
    """Every operator output of one view, as a dict of digests, counts and samples.  `ops` is an operator set with the product's argument
    order (kintinuous_b200.ops, or make_golden's adapter of the reference's operators)."""
    g = {}
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device="cuda")        # noqa: E731
    rows, cols = ROWS, COLS
    from kintinuous_b200 import synth
    intr = np.array(synth.intrinsics(cols, rows), np.float32)
    trunc = trunc_of(V, vs)
    vs = [float(v) for v in vs]
    ts = z((V ** 3,), torch.int16); cs = z((V ** 3 * 4,), torch.uint8)
    ops.init_volume(ts, cs, V)
    poses = [(R, t), perturbed(R, t)]
    ds = z((rows, cols), torch.float32)
    for j, (Rj, tj) in enumerate(poses):
        d, c = _frame(Rj, tj, vs, cols, rows, _render_t(name, V, vs) if j == 0 else None)
        dd = dev(d.view(np.int16)); cc = dev(c)
        fb = z((rows, cols), torch.int16); ops.bilateral(dd, fb, rows, cols)
        vm = z((3 * rows, cols), torch.float32); nm = z((3 * rows, cols), torch.float32)
        ops.create_vmap(intr, fb, vm, rows, cols); ops.create_nmap(vm, nm, rows, cols)
        g[f"nmap_{j}"] = digest.values(nm.cpu().numpy())
        Rinv = np.linalg.inv(Rj.astype(np.float64)).astype(np.float32)
        ops.integrate(dd, rows, cols, intr, vs, Rinv, tj, trunc, ts, cs, V, wrap, cc, nm, 1, ds)
    torch.cuda.synchronize()
    tsdf = ts.cpu().numpy(); col = cs.cpu().numpy().reshape(-1, 4)
    touched = np.flatnonzero(col[:, 3])
    g["touched"] = len(touched)
    g["tsdf"] = digest.raw(tsdf); g["color"] = digest.raw(col)
    idx = touched[sample(len(touched), 400, V)]
    g["vox_idx"] = idx.astype(np.int32); g["vox_tsdf"] = tsdf[idx]; g["vox_color"] = col[idx]
    del tsdf, col
    casts = [(j, rows, cols) for j in range(2)]
    if V in (256, 384) and name in AXIS_VIEWS and vs == [SIZE] * 3:
        casts.append((0, 480, 640))                                          # cx = 320, cy = 267: rays with zero direction components
    for j, r, cl in casts:
        Rj, tj = poses[j]
        tag = f"ray{j}" if r == rows else f"ray{j}_{cl}"
        k = np.array(synth.intrinsics(cl, r), np.float32)
        va = z((3 * r, cl), torch.float32); na = z((3 * r, cl), torch.float32); xa = z((r, cl, 4), torch.uint8)
        ops.raycast(k, Rj, tj, trunc, vs, ts, V, va, na, r, cl, wrap, xa, cs)
        torch.cuda.synchronize()
        v = va.cpu().numpy(); n = na.cpu().numpy(); x = xa.cpu().numpy()
        g[f"{tag}_v"] = digest.vmap(v, r, cl); g[f"{tag}_n"] = digest.vmap(n, r, cl); g[f"{tag}_c"] = digest.raw(x)
        hit = np.flatnonzero(~np.isnan(v.reshape(3, -1)[0]))
        g[f"{tag}_hits"] = len(hit)
        px = hit[sample(len(hit), 60, 7 + j)]
        g[f"{tag}_px"] = px.astype(np.int32); g[f"{tag}_pv"] = v.reshape(3, -1)[:, px]; g[f"{tag}_pc"] = x.reshape(-1, 4)[px]
    out = z((CAP * 32,), torch.uint8)
    for bname, box in slabs(V).items():
        n = ops.extract_slice(ts, vs, V, out, CAP, wrap, cs, box, 1, wrap)
        assert n < CAP, (name, bname, n)
        if getattr(ops, "racy", False):               # the reference's extraction of this slab is not well defined (R1): not recorded
            continue
        g[f"ext_{bname}_n"] = n
        g[f"ext_{bname}"] = digest.raw(digest.canon(out[:n * 32].cpu().numpy().view(np.uint8).reshape(n, 32))) if n else ""
    del out
    for axis, back, cur, delta in clear_runs(V):
        ops.clear_volume(axis, back, ts, cs, V, cur, delta)
    torch.cuda.synchronize()
    g["clear_tsdf"] = digest.raw(ts.cpu().numpy()); g["clear_color"] = digest.raw(cs.cpu().numpy())
    return g


def cleared_planes(ops, torch, V):
    """For every run of clear_runs(V) on a sentinel-filled volume: the storage planes it zeroes (each one whole, in TSDF and colour)."""
    g = {}
    for axis, back, cur, delta in clear_runs(V):
        x = torch.full((V ** 3,), 7, dtype=torch.int16, device="cuda"); y = torch.full((V ** 3 * 4,), 9, dtype=torch.uint8, device="cuda")
        ops.clear_volume(axis, back, x, y, V, cur, delta)
        zt = (x.view(V, V, V) == 0); zc = (y.view(V, V, V, 4) == 0).all(-1)
        assert bool((zt == zc).all())
        ax = {0: (0, 1), 1: (0, 2), 2: (1, 2)}[axis]                          # tensor dims are (z, y, x)
        full = zt.all(dim=ax[1]).all(dim=ax[0]); part = zt.any(dim=ax[1]).any(dim=ax[0])
        assert bool((full == part).all())
        g[f"a{axis}_b{back}_c{cur}_d{delta}"] = torch.nonzero(full).flatten().cpu().numpy().astype(np.int32)
        del x, y
    return g


def run_case(ops, torch, V, vs, names=None):
    """Every view of one (V, volume_size) case as one flat dict (keys '<view>.<output>'), plus the cleared planes ('clear.<run>')."""
    out = {}
    for name, R, t, wrap in views(V, vs):
        if names is not None and name not in names:
            continue
        for k, v in run_view(ops, torch, V, vs, name, R, t, wrap).items():
            out[f"{name}.{k}"] = v
    if tuple(vs) == (SIZE,) * 3:
        for k, v in cleared_planes(ops, torch, V).items():
            out[f"clear.{k}"] = v
    return out


def compare(got, want, prefix=""):
    """Names of the entries of `want` that `got` does not reproduce exactly."""
    bad = []
    for k in want:
        if not k.startswith(prefix):
            continue
        a, b = got.get(k), np.asarray(want[k])
        if a is None or np.asarray(a).shape != b.shape or not np.array_equal(np.asarray(a), b):
            bad.append(k)
    return bad
