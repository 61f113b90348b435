#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the REFERENCE's own CUDA operators (oracle/_ref/libkt_ref_{256,512}.so, built
by oracle/build_ref.sh from the reference sources) on an H100.  The reference ships no golden vectors (SURVEY.md section 4),
so these fixtures are what pins the CPU oracle and the GPU parity tests: they are outputs of the reference itself on seeded
synthetic input.

Run on a GPU machine:   python tools/make_golden.py [OUT]        (writes OUT, default golden_out/, then copy to tests/golden/)
Inputs are re-derivable from kintinuous_b200/synth.py (seed 20260922), so only outputs + a few parameters are stored; outputs
too large to keep are stored as digests (tests/digest.py) or as a seeded sample.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch  # noqa: E402
import digest  # noqa: E402
import kintinuous_b200 as kb  # noqa: E402
from kintinuous_b200 import synth  # noqa: E402
from oracle import refbind  # noqa: E402

OUT = sys.argv[1] if len(sys.argv) > 1 else "golden_out"
V = 256
SIZE = 6.0


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def main():
    os.makedirs(OUT, exist_ok=True)
    ref = refbind.RefCuda(V)
    # ---------------- operator fixtures at 160 x 120 ----------------
    rows, cols = 120, 160
    fx, fy, cx, cy = synth.intrinsics(cols, rows)
    intr = np.array([fx, fy, cx, cy], np.float32)
    depth0, rgb0 = synth.render(0, cols, rows)
    depth3, _ = synth.render(12, cols, rows)          # frame 12 at quarter resolution ~ 3 px of motion
    d0 = dev(depth0.view(np.int16)); d3 = dev(depth3.view(np.int16)); c0 = dev(rgb0)
    g = {}
    fb = torch.zeros_like(d0); ref.bilateral(d0, fb, rows, cols); g["bilateral"] = fb.cpu().numpy().view(np.uint16)
    p1 = torch.zeros((rows // 2, cols // 2), dtype=torch.int16, device="cuda"); ref.pyrdown(fb, p1, rows, cols); g["pyrdown"] = p1.cpu().numpy().view(np.uint16)
    vm = torch.zeros((3 * rows, cols), dtype=torch.float32, device="cuda"); nm = torch.zeros_like(vm)
    ref.vmap(fb, vm, rows, cols, intr); ref.nmap(vm, nm, rows, cols)
    g["vmap"] = vm.cpu().numpy(); g["nmap"] = nm.cpu().numpy()
    R0 = np.eye(3, dtype=np.float32); t0 = np.array([3, 3, 3], np.float32)
    ang = 0.03
    R1 = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], np.float32)
    t1 = t0 + np.array([0.02, -0.01, 0.03], np.float32)
    gv = torch.zeros_like(vm); gn = torch.zeros_like(vm)
    ref.transform_maps(vm, nm, R1, t1, gv, gn, rows, cols); g["transform_v"] = gv.cpu().numpy(); g["transform_n"] = gn.cpu().numpy()
    rv = torch.zeros((3 * rows // 2, cols // 2), dtype=torch.float32, device="cuda"); rn = torch.zeros_like(rv)
    ref.resize_vmap(gv, rv, rows, cols); ref.resize_nmap(gn, rn, rows, cols); g["resize_v"] = rv.cpu().numpy(); g["resize_n"] = rn.cpu().numpy()
    # icp step: model = frame 0 in the volume frame, current = later frame
    mv = torch.zeros_like(vm); mn = torch.zeros_like(vm); ref.transform_maps(vm, nm, R0, t0, mv, mn, rows, cols)
    f3 = torch.zeros_like(d0); ref.bilateral(d3, f3, rows, cols)
    cv = torch.zeros_like(vm); cn = torch.zeros_like(vm); ref.vmap(f3, cv, rows, cols, intr); ref.nmap(cv, cn, rows, cols)
    A, b, res = ref.icp_step(R0, t0, cv, cn, R0, t0, intr, mv, mn, rows, cols)
    g["icp_A"] = A; g["icp_b"] = b; g["icp_res"] = res
    # integrate two frames (second with a wrapped volume and rotated pose), then raycast / extract / clear
    voxel = np.float32(SIZE) / np.float32(V)
    trunc = float(max(np.float32(max(0.01, SIZE / 100.0)), np.float32(2.1) * voxel))
    vs = [SIZE] * 3
    ts = torch.zeros(V ** 3, dtype=torch.int16, device="cuda"); cs = torch.zeros(V ** 3 * 4, dtype=torch.uint8, device="cuda")
    ref.init_volume(ts, cs)
    ds = torch.zeros((rows, cols), dtype=torch.float32, device="cuda")
    wrap = (14, 3, 250)
    ref.integrate(d0, rows, cols, intr, vs, R0, t0, trunc, ts, cs, wrap, c0, nm, 1, ds)
    g["depth_scaled"] = ds.cpu().numpy()
    ref.integrate(d3, rows, cols, intr, vs, np.linalg.inv(R1.astype(np.float64)).astype(np.float32), t1, trunc, ts, cs, wrap, c0, cn, 1, ds)
    torch.cuda.synchronize()
    tsdf = ts.cpu().numpy().reshape(V, V, V); col = cs.cpu().numpy().reshape(V, V, V, 4)
    nz_all = np.flatnonzero(col[..., 3].reshape(-1))              # every voxel ever touched (weight != 0)
    nz = nz_all[::4]                                              # every 4th touched voxel; its own file keeps each fixture under 1 MB
    np.savez_compressed(os.path.join(OUT, "ops_160x120_volume.npz"), vol_touched=np.int64(len(nz_all)), vol_idx=nz.astype(np.int32),
                        vol_tsdf=tsdf.reshape(-1)[nz], vol_color=col.reshape(-1, 4)[nz],
                        vol_tsdf_sha256=np.array(digest.raw(tsdf)), vol_color_sha256=np.array(digest.raw(col)))    # the whole volume, bit for bit
    va = torch.zeros_like(vm); na = torch.zeros_like(vm); cc = torch.zeros((rows, cols, 4), dtype=torch.uint8, device="cuda")
    ref.raycast(intr, R1, t1, trunc, vs, ts, va, na, rows, cols, wrap, cc, cs)
    g["raycast_v"] = va.cpu().numpy(); g["raycast_n"] = na.cpu().numpy(); g["raycast_c"] = cc.cpu().numpy()
    cap = 400000
    ob = torch.zeros(cap * 32, dtype=torch.uint8, device="cuda")
    real = (14, 3, 250 - V)
    for name, box in {"zslab": (0, V, 0, V, 225, 242), "xplus": (0, 120, 0, V, 0, V), "yslab": (0, V, 180, 197, 0, V)}.items():
        n = ref.extract(ts, vs, ob, cap, wrap, cs, box, 1, real)
        pts = ob.cpu().numpy().view(refbind.POINT_DTYPE)[:n]
        arr = np.ascontiguousarray(pts).view(np.uint64).reshape(n, 4)
        g[f"extract_{name}"] = arr[np.lexsort(arr.T[::-1])] if n else arr
    # clear: sentinel-filled volumes, record which storage planes along the axis end up zero
    sent_t = torch.full((V ** 3,), 7, dtype=torch.int16, device="cuda"); sent_c = torch.full((V ** 3 * 4,), 9, dtype=torch.uint8, device="cuda")
    for axis in range(3):
        for back, (cur, n) in ((0, (14, 14)), (1, (-3, -14)), (0, (40, 16)), (1, (5, -16)), (0, (250, 14)), (1, (3, -14)), (0, (-20, 1)), (1, (0, -2))):
            x, y = sent_t.clone(), sent_c.clone()
            ref.clear(axis, back, x, y, cur, cur + n); torch.cuda.synchronize()
            zt = (x.view(V, V, V) == 0); zc = (y.view(V, V, V, 4) == 0).all(-1)
            assert bool((zt == zc).all())
            ax = {0: (0, 1), 1: (0, 2), 2: (1, 2)}[axis]          # tensor dims are (z, y, x)
            full = zt.all(dim=ax[1]).all(dim=ax[0]); part = zt.any(dim=ax[1]).any(dim=ax[0])
            assert bool((full == part).all())                     # planes are cleared completely or not at all
            g[f"clear_a{axis}_b{back}_c{cur}_n{n}"] = torch.nonzero(full).flatten().cpu().numpy().astype(np.int32)
    g["params"] = np.array([rows, cols, V, SIZE, trunc, ang], np.float64)
    np.savez_compressed(os.path.join(OUT, "ops_160x120.npz"), **g)

    # ---------------- RGB-D operator fixtures ----------------
    h = {}
    depth1, rgb1 = synth.render(4, cols, rows)
    d1 = dev(depth1.view(np.int16)); c1 = dev(rgb1)
    fd0 = torch.zeros((rows, cols), dtype=torch.float32, device="cuda"); fd1 = torch.zeros_like(fd0)
    ref.short_depth_to_metres(d0, fd0, rows, cols, 6000); ref.short_depth_to_metres(d1, fd1, rows, cols, 6000)
    i0 = torch.zeros((rows, cols), dtype=torch.uint8, device="cuda"); i1 = torch.zeros_like(i0)
    ref.bgr_to_intensity(c0, i0, rows, cols); ref.bgr_to_intensity(c1, i1, rows, cols)
    h["depth_f"] = fd1.cpu().numpy(); h["intensity"] = i1.cpu().numpy()
    pf = torch.zeros((rows // 2, cols // 2), dtype=torch.float32, device="cuda"); ref.pyrdown_gauss_f(fd1, pf, rows, cols); h["pyr_f"] = pf.cpu().numpy()
    pu = torch.zeros((rows // 2, cols // 2), dtype=torch.uint8, device="cuda"); ref.pyrdown_uchar_gauss(i1, pu, rows, cols); torch.cuda.synchronize(); h["pyr_u"] = pu.cpu().numpy()
    dx = torch.zeros((rows, cols), dtype=torch.int16, device="cuda"); dy = torch.zeros_like(dx)
    ref.derivative_images(i1, dx, dy, rows, cols); h["dIdx"] = dx.cpu().numpy(); h["dIdy"] = dy.cpu().numpy()
    cl = torch.zeros((rows, cols, 3), dtype=torch.float32, device="cuda")
    kd = np.array([float(np.float32(fx)), float(np.float32(fy)), float(np.float32(cx)), float(np.float32(cy))], np.float64)
    ref.project_to_point_cloud(fd0, cl, rows, cols, kd, 0); h["cloud"] = cl.cpu().numpy()
    K = np.array([[kd[0], 0, kd[2]], [0, kd[1], kd[3]], [0, 0, 1]])
    Rw = np.array([[np.cos(0.004), 0, np.sin(0.004)], [0, 1, 0], [-np.sin(0.004), 0, np.cos(0.004)]])
    tw = np.array([-0.01, 0.001, -0.004])
    krk = (K @ Rw @ np.linalg.inv(K)).astype(np.float32); kt = (K @ tw).astype(np.float32)
    cor = torch.zeros(rows * cols * 16, dtype=torch.uint8, device="cuda")
    sigma, count = ref.rgb_residual(float(3.0 ** 2 / (1 / 8.0) ** 2), dx, dy, fd0, fd1, i0, i1, cor, rows, cols, 0.07, kt, krk)
    h["corres"] = cor.cpu().numpy().reshape(rows * cols, 16); h["sigma_count"] = np.array([sigma, count], np.int64)
    h["krk"] = krk; h["kt"] = kt
    sig = float(np.sqrt(count))
    A, b = ref.rgb_step(cor, sig, cl, kd[0], kd[1], dx, dy, 1 / 8.0, rows, cols)
    h["rgb_A"] = A; h["rgb_b"] = b
    np.savez_compressed(os.path.join(OUT, "rgbd_160x120.npz"), **h)

    # before the first full-volume extraction of the process (finalise below): see the NOTE there
    live(ref)

    # ---------------- tracker fixtures: 640x480 into 256^3, three odometry modes + a shifting run ----------------
    rows, cols = 480, 640
    frames = [synth.render(k, cols, rows) for k in range(10)]
    # NOTE the shifting run goes FIRST: the reference's extract kernel publishes its point count from the first warp of the
    # last CTA while other warps may still be appending (extract.cu:290-305), so a full-volume extraction (finalise) can leak a
    # few counts into the NEXT extractCloudSlice call of the same process (observed: 71 phantom points).  DESIGN.md, R1.
    for name, kw in {"icp_shift": dict(odometry=0, voxel_shift=2), "icp": dict(odometry=0), "rgbd": dict(odometry=1), "icp_rgbd": dict(odometry=2)}.items():
        cfg = kb.Config.default(rows=rows, cols=cols, vol=V, **kw)
        rt = ref.tracker(refbind.TrackerConfig.from_kt(cfg))
        poses = []; traces = []
        for k, (d, c) in enumerate(frames):
            rt.process(d, c, k)
            R, t, gcam, w = rt.pose()
            poses.append(np.concatenate([R.reshape(-1), t, gcam, w.astype(np.float32)]))
            if k in (1, 2):
                traces.append(rt.trace())
        ts_, cs_ = rt.export_volume()
        touched = np.flatnonzero(cs_[..., 3].reshape(-1))
        rt.finalise()
        nsl = rt.num_slices()
        sl = [(rt.get_slice(i)[1], len(rt.get_slice(i)[0])) for i in range(nsl)]
        np.savez_compressed(os.path.join(OUT, f"tracker_{name}_256.npz"), poses=np.array(poses, np.float32), trace1=traces[0], trace2=traces[1],
                            touched=np.int64(len(touched)), tsdf_hist=np.bincount((ts_.reshape(-1)[touched].astype(np.int32) + 32768) >> 8, minlength=256),
                            weight_hist=np.bincount(cs_[..., 3].reshape(-1)[touched], minlength=256), slices=np.array(sl, np.int64).reshape(-1, 2))
        print(name, "done; slices", sl, flush=True)
        rt.close()
    print("golden written to", OUT)


# ---------------- fixtures of the GPU parity tests that compare with the reference's CUDA path ----------------
def _sample(n, k, seed):
    """k of n indices, sorted, seeded: the tests draw the same ones."""
    return np.sort(np.random.default_rng(seed).choice(n, size=min(k, n), replace=False))


def _z(shape, dt):
    return torch.zeros(shape, dtype=dt, device="cuda")


def live(ref):
    """Outputs of the reference's CUDA path for the tests that used to run it next to the product (tests/test_gpu_ops.py,
    test_gpu_tracker.py, test_gpu_baseline_configs.py): each function below runs the reference side of one such test."""
    ops_640(ref)
    image_160(ref)
    wrap_160(ref)
    tracker_live_256(ref)
    for odometry, nframes in ((0, 72), (2, 22), (1, 26)):
        baseline_512(odometry, nframes)


def _front(ref, dd, rows, cols, intr):
    fb = _z((rows, cols), torch.int16); ref.bilateral(dd, fb, rows, cols)
    vm = _z((3 * rows, cols), torch.float32); nm = torch.zeros_like(vm)
    ref.vmap(fb, vm, rows, cols, intr); ref.nmap(vm, nm, rows, cols)
    return fb, vm, nm


def ops_640(ref):
    """test_bilateral_full_resolution_vs_reference and test_volume_ops_vs_reference_cuda_on_identical_buffers (640x480)."""
    g = {}
    rng = np.random.default_rng(20260922)
    inputs = [synth.render(k)[0] for k in (0, 7)]
    noisy = inputs[0].astype(np.int64) + rng.integers(-40, 41, inputs[0].shape)
    noisy[rng.random(noisy.shape) < 0.05] = 0
    inputs.append(np.clip(noisy, 0, 65535).astype(np.uint16))
    far = inputs[0].copy()
    far[100:140, 200:300] = 65535; far[300:330, 10:50] = 50000; far[0:8, 600:640] = 47000
    inputs.append(far)
    inputs.append(rng.integers(0, 65536, inputs[0].shape).astype(np.uint16))
    for i, d in enumerate(inputs):
        b = _z((480, 640), torch.int16); ref.bilateral(dev(d.view(np.int16)), b, 480, 640)
        g[f"bilateral_{i}"] = np.array(digest.raw(b.cpu().numpy()))
        src = b
        for l in range(1, 4):
            r, c = 480 >> (l - 1), 640 >> (l - 1)
            pb = _z((r // 2, c // 2), torch.int16); ref.pyrdown(src, pb, r, c)
            g[f"pyrdown_{i}_{l}"] = np.array(digest.raw(pb.cpu().numpy()))
            src = pb
    rows, cols = 480, 640
    intr = np.array(synth.intrinsics(cols, rows), np.float32)
    d, c = synth.render(3)
    dd = dev(d.view(np.int16)); cc = dev(c)
    fb, vm, nm = _front(ref, dd, rows, cols, intr)
    g["nmap"] = np.array(digest.values(nm.cpu().numpy()))
    tb = _z((V ** 3,), torch.int16); cb = _z((V ** 3 * 4,), torch.uint8); dsb = _z((rows, cols), torch.float32)
    R0 = np.eye(3, dtype=np.float32); t0 = np.array([3, 3, 3], np.float32)
    ang = 0.03
    R1 = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], np.float32)
    t1 = t0 + np.array([0.02, -0.01, 0.03], np.float32)
    voxel = np.float32(SIZE) / np.float32(V)
    trunc = float(max(np.float32(max(0.01, SIZE / 100.0)), np.float32(2.1) * voxel))
    vs = [SIZE] * 3
    for j, (wrap, R, tt) in enumerate([((0, 0, 0), R0, t0), ((250, 14, 3), R1, t1), ((250, 14, 3), R1.T.copy(), t1 + np.float32(0.05))]):
        Rinv = np.linalg.inv(R.astype(np.float64)).astype(np.float32)
        ref.integrate(dd, rows, cols, intr, vs, Rinv, tt, trunc, tb, cb, wrap, cc, nm, 1, dsb)
        torch.cuda.synchronize()
        g[f"vol_tsdf_{j}"] = np.array(digest.raw(tb.cpu().numpy())); g[f"vol_color_{j}"] = np.array(digest.raw(cb.cpu().numpy()))
        vb = _z((3 * rows, cols), torch.float32); nb = _z((3 * rows, cols), torch.float32); xb = _z((rows, cols, 4), torch.uint8)
        ref.raycast(intr, R, tt, trunc, vs, tb, vb, nb, rows, cols, wrap, xb, cb)
        torch.cuda.synchronize()
        g[f"ray_v_{j}"] = np.array(digest.vmap(vb.cpu().numpy(), rows, cols)); g[f"ray_n_{j}"] = np.array(digest.vmap(nb.cpu().numpy(), rows, cols))
        g[f"ray_c_{j}"] = np.array(digest.raw(xb.cpu().numpy()))
    np.savez_compressed(os.path.join(OUT, "ref_ops_640x480.npz"), **g)


def image_160(ref):
    """test_generate_image_and_depth_vs_reference_cuda: the reference's ray-cast surface (the input both sides get) and its images."""
    rows, cols = 120, 160
    intr = np.array(synth.intrinsics(cols, rows), np.float32)
    d, c = synth.render(0, cols, rows)
    dd = dev(d.view(np.int16)); cc = dev(c)
    fb, vm, nm = _front(ref, dd, rows, cols, intr)
    ts = _z((V ** 3,), torch.int16); cs = _z((V ** 3 * 4,), torch.uint8); ds = _z((rows, cols), torch.float32)
    R = np.eye(3, dtype=np.float32); t = np.array([3, 3, 3], np.float32)
    for _ in range(3):
        ref.integrate(dd, rows, cols, intr, [6.0] * 3, R, t, 0.06, ts, cs, (0, 0, 0), cc, nm, 1, ds)
    ang = 0.02
    R1 = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], np.float32)
    t1 = t + np.array([0.01, 0.0, 0.02], np.float32)
    va = torch.zeros_like(vm); na = torch.zeros_like(vm); xa = _z((rows, cols, 4), torch.uint8)
    ref.raycast(intr, R1, t1, 0.06, [6.0] * 3, ts, va, na, rows, cols, (0, 0, 0), xa, cs)
    light = [-18.0, -18.0, -18.0]
    ib = _z((rows, cols, 3), torch.uint8); cb = torch.zeros_like(ib)
    ref.generate_image(va, na, xa, light, 1, ib, cb, rows, cols)
    Rinv = np.linalg.inv(R1.astype(np.float64)).astype(np.float32)
    db = _z((rows, cols), torch.int16)
    ref.generate_depth(Rinv, t1, va, na, db, rows, cols)
    torch.cuda.synchronize()
    np.savez_compressed(os.path.join(OUT, "ref_image_160x120.npz"), vmap=va.cpu().numpy(), nmap=na.cpu().numpy(), vmap_color=xa.cpu().numpy(),
                        image=ib.cpu().numpy(), image_color=cb.cpu().numpy(), depth=db.cpu().numpy())


def wrap_160(ref):
    """test_wrap_beyond_one_volume_length: integrate, raycast, extract, clear at voxel offsets beyond one volume length."""
    g = {}
    rows, cols = 120, 160
    intr = np.array(synth.intrinsics(cols, rows), np.float32)
    d, c = synth.render(0, cols, rows)
    dd = dev(d.view(np.int16)); cc = dev(c)
    fb, vm, nm = _front(ref, dd, rows, cols, intr)
    g["nmap"] = np.array(digest.values(nm.cpu().numpy()))
    vs = [SIZE] * 3; trunc = 0.06
    ang = 0.05
    R = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], np.float32)
    Rinv = np.linalg.inv(R.astype(np.float64)).astype(np.float32)
    t = np.array([3.02, 2.99, 3.01], np.float32)
    for i, wrap in enumerate(((V + 88, 2 * V + 3, 3 * V - 1), (V, 2 * V, 0), (5 * V + 17, 31, V + 200))):
        tb = _z((V ** 3,), torch.int16); cb = _z((V ** 3 * 4,), torch.uint8); ds = _z((rows, cols), torch.float32)
        ref.integrate(dd, rows, cols, intr, vs, Rinv, t, trunc, tb, cb, wrap, cc, nm, 1, ds)
        torch.cuda.synchronize()
        g[f"tsdf_{i}"] = np.array(digest.raw(tb.cpu().numpy())); g[f"color_{i}"] = np.array(digest.raw(cb.cpu().numpy()))
        vb = torch.zeros_like(vm); nb = torch.zeros_like(vm); xb = _z((rows, cols, 4), torch.uint8)
        ref.raycast(intr, R, t, trunc, vs, tb, vb, nb, rows, cols, wrap, xb, cb)
        torch.cuda.synchronize()
        g[f"ray_v_{i}"] = np.array(digest.raw(vb.cpu().numpy())); g[f"ray_n_{i}"] = np.array(digest.raw(nb.cpu().numpy()))
        g[f"ray_c_{i}"] = np.array(digest.raw(xb.cpu().numpy()))
        cap = 400000
        ob = _z((cap * 32,), torch.uint8)
        n_b = ref.extract(tb, vs, ob, cap, wrap, cb, (0, V, 0, V, 225, 242), 1, tuple(int(w) for w in wrap))
        g[f"extract_n_{i}"] = np.int64(n_b)
        g[f"extract_{i}"] = np.array(digest.raw(digest.canon(ob.cpu().numpy().view(refbind.POINT_DTYPE)[:n_b])))
        for axis in range(3):
            ref.clear(axis, 0, tb, cb, wrap[axis], wrap[axis] + 14)
        torch.cuda.synchronize()
        g[f"clear_tsdf_{i}"] = np.array(digest.raw(tb.cpu().numpy())); g[f"clear_color_{i}"] = np.array(digest.raw(cb.cpu().numpy()))
    np.savez_compressed(os.path.join(OUT, "ref_wrap_160x120.npz"), **g)


def _pose_row(t):
    R, tt, gc, w = t.pose()
    return np.concatenate([R.reshape(-1), tt, gc]).astype(np.float32), w.astype(np.int32)


def tracker_live_256(ref):
    """test_tracker_vs_reference_cuda_live and test_degenerate_frames_vs_reference_cuda_live: the reference tracker's poses, a seeded
    sample of its fused volume, and its model maps."""
    frames = [synth.render(k) for k in range(10)]
    cfg = kb.Config.default(vol=V)
    rt = ref.tracker(refbind.TrackerConfig.from_kt(cfg))
    g = {}
    P = []; W = []
    for k, (d, c) in enumerate(frames):
        rt.process(d, c, k); p, w = _pose_row(rt); P.append(p); W.append(w)
    g["poses"] = np.array(P); g["wraps"] = np.array(W)
    tb, cb = rt.export_volume()
    touched = np.flatnonzero(cb[..., 3].reshape(-1))
    g["touched"] = np.int64(len(touched))
    idx = touched[_sample(len(touched), 50000, 1)]
    g["vol_idx"] = idx.astype(np.int32); g["vol_tsdf"] = tb.reshape(-1)[idx]; g["vol_weight"] = cb[..., 3].reshape(-1)[idx]
    for lvl in range(3):
        vb = rt.download_map(2, lvl)
        nan = np.isnan(vb[0])
        g[f"map_nan_{lvl}"] = np.packbits(nan.reshape(-1))
        px = np.flatnonzero(~nan.reshape(-1))
        px = px[_sample(len(px), 5000, 2 + lvl)]
        g[f"map_px_{lvl}"] = px.astype(np.int32); g[f"map_v_{lvl}"] = vb.reshape(3, -1)[:, px]
    rt.close()
    np.savez_compressed(os.path.join(OUT, "ref_tracker_live_256.npz"), **g)

    h = {}
    rng = np.random.default_rng(11)
    seq = []
    for k in range(8):
        d, c = synth.render(k, noise=True) if k in (1, 2) else frames[k]
        d = d.copy()
        if k == 3:
            d[:] = 0
        if k == 4:
            d[:, 320:] = 0
        if k == 5:
            d[rng.random(d.shape) < 0.3] = 0
        if k == 6:
            d, c = seq[-1]
        seq.append((d, c))
    for odometry in (0, 2):
        rt = ref.tracker(refbind.TrackerConfig.from_kt(kb.Config.default(vol=V, odometry=odometry)))
        P = []; W = []
        for k, (d, c) in enumerate(seq):
            rt.process(d, c, k); p, w = _pose_row(rt); P.append(p); W.append(w)
        h[f"poses_{odometry}"] = np.array(P); h[f"wraps_{odometry}"] = np.array(W)
        if odometry == 0:
            tb, cb = rt.export_volume()
            touched = np.flatnonzero(cb[..., 3].reshape(-1))
            h["touched"] = np.int64(len(touched))
            idx = touched[_sample(len(touched), 100000, 5)]
            h["vol_idx"] = idx.astype(np.int32); h["vol_tsdf"] = tb.reshape(-1)[idx]
        rt.close()
    np.savez_compressed(os.path.join(OUT, "ref_degenerate_256.npz"), **h)


def baseline_512(odometry, nframes):
    """test_baseline_config_512_live_replay_exact: BASELINE configs 1-2 (640x480 into 512^3, -t 14).  Records the reference tracker
    (and, ICP-only, its twin fed a 1-LSB perturbed frame 1), the reference operators' front end of every frame, and the replay of the
    PRODUCT's integration poses through the reference's operators: slices at every shift, the back-wall slab, the final volume."""
    W512 = 512
    ROWS, COLS = 480, 640
    ref = refbind.RefCuda(W512)
    from concurrent.futures import ProcessPoolExecutor
    with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        frames = list(ex.map(synth.render, range(nframes), chunksize=2))
    cfg = kb.Config.default(vol=W512, odometry=odometry)
    mine = kb.Tracker(cfg)
    rt = ref.tracker(refbind.TrackerConfig.from_kt(cfg))
    rp = ref.tracker(refbind.TrackerConfig.from_kt(cfg)) if odometry == 0 else None
    intr = np.array(synth.intrinsics(COLS, ROWS), np.float32)
    vs = [SIZE] * 3
    g = {"trunc": np.float32(rt.trunc_dist)}
    trunc = mine.trunc_dist
    ts = _z((W512 ** 3,), torch.int16); cs = _z((W512 ** 3 * 4,), torch.uint8)
    ref.init_volume(ts, cs)
    fb = _z((ROWS, COLS), torch.int16); vm = _z((3 * ROWS, COLS), torch.float32); nm = torch.zeros_like(vm); ds = _z((ROWS, COLS), torch.float32)
    cap = 3 * ROWS * COLS
    ob = _z((cap * 32,), torch.uint8)
    cur = [0, 0, 0]
    P, W, PP, WP, FB, VM, NM, INTEG = [], [], [], [], [], [], [], []
    sl = []
    for k in range(nframes):
        d, c = frames[k]
        pm = mine.process_frame(d, c, k); rt.process(d, c, k)
        p, w = _pose_row(rt); P.append(p); W.append(w)
        if rp is not None:
            dp = d
            if k == 1:
                dp = d.copy(); dp[ROWS // 2, COLS // 2] += 1
            rp.process(dp, c, k)
            p, w = _pose_row(rp); PP.append(p); WP.append(w)
        dd = dev(d.view(np.int16)); cc = dev(c)
        ref.bilateral(dd, fb, ROWS, COLS); ref.vmap(fb, vm, ROWS, COLS, intr); ref.nmap(vm, nm, ROWS, COLS)
        FB.append(digest.raw(fb.cpu().numpy().view(np.uint16)))
        VM.append(digest.values(vm.cpu().numpy().reshape(3, ROWS, COLS))); NM.append(digest.values(nm.cpu().numpy().reshape(3, ROWS, COLS)))
        wa = pm.as_tuple()[3]
        for axis in range(3):
            n = int(wa[axis]) - cur[axis]
            if n == 0:
                continue
            lo, hi = [0, 0, 0], [W512, W512, W512]
            if n > 0:
                lo[axis], hi[axis] = 0, n + 1 + cfg.overlap
            elif axis < 2:
                lo[axis], hi[axis] = W512 + (n - cfg.overlap), W512
            else:
                lo[axis], hi[axis] = W512 + (n - cfg.overlap) - 1, W512 - 1
            box = (lo[0], hi[0], lo[1], hi[1], lo[2], hi[2])
            vw = [int(x) if x >= 0 else W512 - ((-int(x)) % W512) for x in cur]
            cnt = ref.extract(ts, vs, ob, cap, vw, cs, box, 1, cur)
            sl.append((k, axis, n, cnt, digest.raw(digest.canon(ob.cpu().numpy().view(refbind.POINT_DTYPE)[:cnt]))))
            ref.clear(axis, 1 if n < 0 else 0, ts, cs, cur[axis], cur[axis] + n)
            cur[axis] += n
        Rinv, tint, wint = mine.last_integrate()
        INTEG.append(digest.raw(np.concatenate([Rinv.reshape(-1), tint, wint.astype(np.float32)])))
        ref.integrate(dd, ROWS, COLS, intr, vs, Rinv, tint, trunc, ts, cs, wint, cc, nm, 1, ds)
    g["poses"] = np.array(P); g["wraps"] = np.array(W)
    if rp is not None:
        g["poses_perturbed"] = np.array(PP); g["wraps_perturbed"] = np.array(WP)
    g["bilateral"] = np.array(FB); g["vmap"] = np.array(VM); g["nmap"] = np.array(NM); g["integrate_pose"] = np.array(INTEG)
    g["slice_events"] = np.array([s[:4] for s in sl], np.int64).reshape(-1, 4); g["slice_points"] = np.array([s[4] for s in sl])
    if odometry == 0:
        wall = int((5.5 - cur[2] * SIZE / W512) / (SIZE / W512))
        box = (0, W512, 0, W512, max(0, wall - 15), min(W512 - 1, wall + 15))
        vw = [int(x) if x >= 0 else W512 - ((-int(x)) % W512) for x in cur]
        n_b = ref.extract(ts, vs, ob, cap, vw, cs, box, 1, cur)
        g["wall_box"] = np.array(box, np.int64); g["wall_n"] = np.int64(n_b)
        g["wall_points"] = np.array(digest.raw(digest.canon(ob.cpu().numpy().view(refbind.POINT_DTYPE)[:n_b])))
    rs = [(rt.get_slice(i)[1], len(rt.get_slice(i)[0])) for i in range(rt.num_slices())]
    g["ref_slices"] = np.array(rs, np.int64).reshape(-1, 2)
    torch.cuda.synchronize()
    tr_ = ts.cpu().numpy(); cr_ = cs.cpu().numpy().reshape(-1, 4)
    g["replay_tsdf"] = np.array(digest.raw(tr_)); g["replay_color"] = np.array(digest.raw(cr_)); g["replay_touched"] = np.int64((cr_[:, 3] != 0).sum())
    tb_, cb_ = rt.export_volume()
    touched = np.flatnonzero(cb_[..., 3].reshape(-1))
    idx = touched[_sample(len(touched), 50000, 7)]
    g["ref_vol_idx"] = idx.astype(np.int32); g["ref_vol_tsdf"] = tb_.reshape(-1)[idx]
    mine.close(); rt.close()
    if rp is not None:
        rp.close()
    np.savez_compressed(os.path.join(OUT, f"ref_baseline_512_odo{odometry}.npz"), **g)
    print("baseline", odometry, "slices", len(sl), flush=True)


if __name__ == "__main__":
    main()
