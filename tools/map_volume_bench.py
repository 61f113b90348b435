"""What the map volume costs (kt_mapvol.cu), as one JSON line.

  store: the synthetic stream (640x480, voxel shift 2) tracked at 512^3 and 1024^3 with the map volume off, on, and on with restore;
         the frame time is a host clock around each frame, which ends in a synchronise.  Shift frames carry the store's three launches
         per cleared slab (four with restore), so the difference of their medians is what a shift costs; frames without a shift should
         not change.
  drift: a noisy out-and-back stream (640x480 into 128^3 and 256^3 over 3 m, voxel shift 2, 0.025 m per frame along +-x, +-y, +-z) tracked with
         the map volume on, restore off and on: the translation error against the rendered ground truth per frame, its maximum, and
         at each return to the start.
  export: kt_op_mesh_bricks over every brick with a surface voxel of a sphere in a 1024^3 grid, CUDA events around the call.

Usage: python tools/map_volume_bench.py [--frames 120] [--repeat 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception:
        return "unknown"


def tracker_cost(kb, vol, frames, store, restore=False):
    """Frame times (ms, host clock around each synchronous frame) and launches of the shifting stream, store on or off, restore on or off."""
    from kintinuous_b200 import synth
    rows, cols = 480, 640
    trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=vol, odometry=0, voxel_shift=2))
    if store:
        trk.set_map_volume(True, 1 << 20)
        trk.set_map_volume_restore(restore)
    seq = [synth.render(k, cols, rows) for k in range(frames)]
    times, shift_times, launches = [], [], 0
    for k, (d, c) in enumerate(seq):
        l0 = trk.launch_count()
        t0 = time.perf_counter()
        p = trk.process_frame(d, c, k)
        trk.pose()
        dt = (time.perf_counter() - t0) * 1e3
        launches += trk.launch_count() - l0
        (shift_times if p.shifted else times).append(dt)
    info = trk.map_volume_info() if store else (0, 0, False)
    gm = trk.global_mesh(8)[2] if store else None
    trk.close()
    return {"frame_ms_median": float(np.median(times)), "shift_frame_ms_median": float(np.median(shift_times)) if shift_times else None,
            "shift_frames": len(shift_times), "launches": launches, "bricks": int(info[0]), "brick_mb": info[0] * 3072 / 2 ** 20,
            "export": gm}


def drift(kb, restore, vol, leg=20, step=0.025):
    """Per-frame translation error (m) of the noisy out-and-back stream against its ground truth, restore off or on.  The tracked
    position is the volume-relative translation plus the voxel wrap."""
    from kintinuous_b200 import synth
    rows, cols = 480, 640
    trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=vol, volume_size=3.0, odometry=0, voxel_shift=2))
    trk.set_map_volume(True, 1 << 16)
    trk.set_map_volume_restore(restore)
    steps, traj = np.zeros(3, np.int64), [np.zeros(3, np.int64)]
    for axis, sgn in ((0, 1), (0, -1), (1, 1), (1, -1), (2, 1), (2, -1)):
        for _ in range(leg):
            steps = steps.copy(); steps[axis] += sgn
            traj.append(steps)
    err, p0 = [], None
    for k, s in enumerate(traj):
        d, c = synth.render_at(np.eye(3), s * step, cols, rows, noise=True, noise_seed=k)
        p = trk.process_frame(d, c, k)
        pos = np.array(p.t, np.float64) + np.array(p.voxel_wrap, np.float64) * trk.voxel_size
        p0 = pos if p0 is None else p0
        err.append(float(np.linalg.norm((pos - p0) - s * step)))
    trk.close()
    home = [k for k in range(1, len(traj)) if not traj[k].any()]
    return {"frames": len(traj), "err_m": [round(e, 6) for e in err], "err_max_m": max(err), "err_at_start_m": {str(k): err[k] for k in home}}


def export_cost(kb, torch, repeat):
    N, size = 1024, 6.0
    ar = torch.arange(N, device="cuda", dtype=torch.float32)
    z, y, x = ar.view(N, 1, 1), ar.view(1, N, 1), ar.view(1, 1, N)
    d = torch.sqrt((x - 0.5 * N) ** 2 + (y - 0.5 * N) ** 2 + (z - 0.5 * N) ** 2) - 0.4 * N
    tsdf = torch.trunc(torch.clamp(d / 4.0, -1, 1) * 32767).to(torch.int16)
    del d
    col = torch.full((N, N, N, 4), 20, dtype=torch.uint8, device="cuda")
    nb = N // 8
    bt = tsdf.view(nb, 8, nb, 8, nb, 8).permute(0, 2, 4, 1, 3, 5).reshape(-1, 8, 8, 8)
    keep = (bt != 32767).flatten(1).any(-1)
    bz, by, bx = torch.meshgrid(*[torch.arange(nb, device="cuda", dtype=torch.int64)] * 3, indexing="ij")
    bias = 1 << 20
    keys = (((bz + bias) << 42) | ((by + bias) << 21) | (bx + bias)).flatten()[keep].contiguous()
    bt = bt[keep].contiguous()
    bc = col.view(nb, 8, nb, 8, nb, 8, 4).permute(0, 2, 4, 1, 3, 5, 6).reshape(-1, 8, 8, 8, 4)[keep].contiguous()
    del tsdf, col
    _, nv, nt = kb.ops.mesh_bricks_into(keys, bt, bc, len(keys), [size] * 3, N, 8, None, 0, None, 0)
    v = torch.empty(nv * 32, dtype=torch.uint8, device="cuda"); t = torch.empty(nt * 12, dtype=torch.uint8, device="cuda")
    ms = []
    for _ in range(repeat + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        kb.ops.mesh_bricks_into(keys, bt, bc, len(keys), [size] * 3, N, 8, v, nv, t, nt)
        e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return {"bricks": int(len(keys)), "verts": nv, "tris": nt, "ms_median": float(np.median(ms[1:])), "ms_first": ms[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    import torch
    import kintinuous_b200 as kb
    if not kb.cuda_available():
        raise SystemExit("map_volume_bench: no CUDA device")
    out = {"gpu": _gpu()}
    for vol in (512, 1024):
        out[f"tracker_{vol}"] = {"off": tracker_cost(kb, vol, a.frames, False), "on": tracker_cost(kb, vol, a.frames, True),
                                 "on_restore": tracker_cost(kb, vol, a.frames, True, True)}
    for vol in (128, 256):
        out[f"drift_out_and_back_{vol}"] = {"restore_off": drift(kb, False, vol), "restore_on": drift(kb, True, vol)}
    out["export_1024_sphere"] = export_cost(kb, torch, a.repeat)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
