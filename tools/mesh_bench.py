#!/usr/bin/env python3
"""Cost of the marching-cubes mesher (kt_mesh.cu) on the baseline workload: 640x480 synthetic frames into a 512^3 volume.

Prints one JSON line with
  * kt_op_mesh_volume over the whole volume after the 72-frame sequence: median / min / max of CUDA-event times over --calls warm calls,
    vertex and triangle counts, and that time against reading the 2-byte TSDF plane once at the data-sheet HBM3 bandwidth (268 MB at
    3.35 TB/s = 80 us: a floor, not a target);
  * the same operator on one shift slab (17 planes of 512^2: voxel_shift 14 + 1 + overlap 2), i.e. what meshing adds to a shifting frame:
    the +x slab that leaves next (empty of surface in this trajectory) and, for scale, a 17-plane slab through the middle of the scene;
  * frames/s of the 72-frame shifting sequence with slice meshing on and off, alternating in this one process, --reps runs each;
  * the GPU's name, power limit and SM clock, read in the same run.
The volume is the tracker's own, exported and re-uploaded, so the timed calls see exactly the tracker's TSDF."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_facts():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smmax = [s.strip() for s in out.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock=sm, sm_clock_max=smmax)
    except Exception as e:                                         # the measurement stands without these, say so
        return dict(gpu="not read: %s" % e)


def run_sequence(kb, frames, mesh):
    trk = kb.Tracker(kb.Config.default(rows=480, cols=640, vol=512, odometry=0))
    if mesh:
        trk.set_slice_meshing(True, 8)
    trk.process_frame(*frames[0], 0)
    trk.span_mark(0)
    for k in range(1, len(frames)):
        trk.process_frame(*frames[k], k)
    trk.span_mark(1)
    ms = trk.span_elapsed_ms()
    return trk, (len(frames) - 1) / (ms / 1e3)


def time_op(kb, torch, td, cd, wrap, box, calls, vbuf, tbuf):
    for _ in range(5):
        kb.ops.mesh_volume_into(td, cd, 512, [6.0] * 3, wrap, wrap, box, 8, vbuf, vbuf.numel() // 32, tbuf, tbuf.numel() // 12)
    t = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        st, nv, nt = kb.ops.mesh_volume_into(td, cd, 512, [6.0] * 3, wrap, wrap, box, 8, vbuf, vbuf.numel() // 32, tbuf, tbuf.numel() // 12)
        e1.record(); e1.synchronize()
        assert st == 0
        t.append(e0.elapsed_time(e1))
    return dict(median_ms=float(np.median(t)), min_ms=float(np.min(t)), max_ms=float(np.max(t)), calls=calls, n_verts=nv, n_tris=nt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=72)
    ap.add_argument("--calls", type=int, default=60)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    if not kb.cuda_available():
        raise SystemExit("mesh_bench: no CUDA device")
    facts = gpu_facts()
    frames = [synth.render(k, 640, 480) for k in range(a.frames)]
    fps = {"on": [], "off": []}
    trk = None
    for r in range(a.reps):
        for mode in (("off", "on") if r % 2 == 0 else ("on", "off")):
            t, f = run_sequence(kb, frames, mode == "on")
            fps[mode].append(f)
            if trk is None and mode == "off":
                trk = t
            else:
                t.close()
    tsdf, col = trk.export_volume()
    wrap = [int(w) for w in trk.pose().voxel_wrap]              # the next +x shift slab is logical [0, 17) at the tracker's wrap
    trk.close()
    td, cd = torch.from_numpy(tsdf).cuda(), torch.from_numpy(col).cuda()
    st, nv, nt = kb.ops.mesh_volume_into(td, cd, 512, [6.0] * 3, wrap, wrap, (0, 512, 0, 512, 0, 512), 8, None, 0, None, 0)
    vbuf = torch.empty(max(nv, 1) * 32, dtype=torch.uint8, device="cuda")
    tbuf = torch.empty(max(nt, 1) * 12, dtype=torch.uint8, device="cuda")
    whole = time_op(kb, torch, td, cd, wrap, (0, 512, 0, 512, 0, 512), a.calls, vbuf, tbuf)
    floor_us = 512 ** 3 * 2 / 3.35e12 * 1e6
    whole["tsdf_read_floor_us"] = round(floor_us, 1)
    whole["time_over_floor"] = round(whole["median_ms"] * 1e3 / floor_us, 1)
    slab = time_op(kb, torch, td, cd, wrap, (0, 17, 0, 512, 0, 512), a.calls, vbuf, tbuf)
    mid = time_op(kb, torch, td, cd, wrap, (247, 264, 0, 512, 0, 512), a.calls, vbuf, tbuf)      # a slab through the scene
    facts["sm_clock_after"] = gpu_facts().get("sm_clock")
    res = dict(metric="mesh_bench", workload="640x480 synth, 512^3, %d frames" % a.frames, **facts,
               mesh_volume_whole=whole, mesh_volume_shift_slab_17=slab, mesh_volume_mid_slab_17=mid,
               fps_meshing_off=[round(x, 1) for x in fps["off"]], fps_meshing_on=[round(x, 1) for x in fps["on"]],
               fps_off_median=round(float(np.median(fps["off"])), 1), fps_on_median=round(float(np.median(fps["on"])), 1),
               timestamp=time.strftime("%Y-%m-%dT%H:%M:%S"))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
