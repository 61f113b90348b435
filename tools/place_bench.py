"""Cost of loop detection on the GPU (kt_op_surf, kt_op_match_ratio, kt_detect_loops) and its effect on tracking throughput.

Prints one JSON line: the GPU's name and power limit read in the same run, then
  surf_ms          one kt_op_surf call on a 640x480 frame (1000 features), CUDA events around it, median of --reps after a warm-up
                   call: the launches plus the call's 4-byte count read-back and stream synchronisation (no allocation: the operator's
                   scratch persists between calls)
  retrieval        per database size K keyframes x 1000 features against 1000 query features: one kt_op_match_ratio call (K segments,
                   the per-keyframe pass counts read back), CUDA events, median of --reps after a warm-up call -- the launches plus the
                   call's small uploads / read-back and synchronisation --, and K * 1000 * 1000 * 64 * 2 FLOP over it (the FFMA count of the
                   distances; each also costs a subtraction, not counted)
  detect_ms_per_keyframe / stages   kt_detect_loops over the keyframes of a 640x480 trajectory that leaves its start and returns,
                   one keyframe per call (host clock around the call, which synchronises): the mean, and how many keyframes ended at
                   each stage
  verify_ms        median time of the keyframes that reached the dense check (retrieval, 3-D matching, PnP, front end + ICP of both
                   keyframes, fitness); "not measured" when none did
  fps_off / fps_on frames/s of the same pre-rendered sequence through kt_process_frame with detection off / on (host clock, ends
                   with a device synchronise; detection's capture runs on its side stream)
Needs a CUDA device: there is no CPU path."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _events_ms(fn, reps):
    import torch
    ts = []
    for _ in range(reps):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def _loop_poses(n_out, stay):
    out = []
    for k in range(2 * n_out + stay):
        s = k if k <= n_out else max(0, 2 * n_out - k)
        a = np.deg2rad(0.6 * s)
        out.append((np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]]), np.array([0.010 * s, 0.0, 0.004 * s])))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", default="100,1000,4000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--vol", type=int, default=512)
    a = ap.parse_args()
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("place_bench: no CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": smi.splitlines()[0] if smi else "unknown"}
    rows, cols = 480, 640
    poses = _loop_poses(60, 10)
    frames = [synth.render_at(R, t, cols, rows, noise=True, noise_seed=k, texture=synth.cell_texture) for k, (R, t) in enumerate(poses)]

    # SURF
    rgb = torch.from_numpy(frames[0][1]).cuda()
    kb.ops.surf(rgb, rows, cols, 1000)
    out["surf_ms"] = _events_ms(lambda: kb.ops.surf(rgb, rows, cols, 1000), a.reps)
    out["surf_features"] = int(len(kb.ops.surf(rgb, rows, cols, 1000)[0]))

    # retrieval
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.randn(1000, 64, device="cuda", generator=g); q /= q.norm(dim=1, keepdim=True)
    out["retrieval"] = []
    for K in [int(s) for s in a.keyframes.split(",")]:
        db = torch.randn(K * 1000, 64, device="cuda", generator=g); db /= db.norm(dim=1, keepdim=True)
        best = torch.empty(K * 1000, dtype=torch.int32, device="cuda"); d1 = torch.empty(K * 1000, device="cuda")
        d2 = torch.empty(K * 1000, device="cuda"); ps = torch.empty(K * 1000, dtype=torch.uint8, device="cuda")
        lib = kb.load()
        import ctypes as C
        sp = np.zeros(K, np.int32)
        call = lambda: lib.kt_op_match_ratio(C.c_void_p(db.data_ptr()), K, 1000, None, C.c_void_p(q.data_ptr()), 1000, C.c_float(0.49),
                                             C.c_void_p(best.data_ptr()), C.c_void_p(d1.data_ptr()), C.c_void_p(d2.data_ptr()), C.c_void_p(ps.data_ptr()),
                                             sp.ctypes.data_as(C.c_void_p), None)
        assert call() == 0
        ms = _events_ms(call, a.reps)
        flop = K * 1000 * 1000 * 64 * 2
        out["retrieval"].append({"keyframes": K, "ms": ms, "tflops": flop / (ms * 1e-3) / 1e12})
        del db, best, d1, d2, ps

    # sequence with detection off / on, then kt_detect_loops
    def run(detect, seq):
        cfg = kb.Config.default(rows=rows, cols=cols, vol=a.vol)
        trk = kb.Tracker(cfg)
        if detect:
            trk.set_loop_detection(True, exclude_recent=3, loop_throttle_s=0.0, close=0)
        trk.process_frame(seq[0][0], seq[0][1], 33333)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(1, len(seq)):
            trk.process_frame(seq[k][0], seq[k][1], 33333 * (k + 1))
        torch.cuda.synchronize()
        fps = (len(seq) - 1) / (time.perf_counter() - t0)
        return trk, fps
    run(False, frames[:5])[0].close()
    trk_off, fps_off = run(False, frames)
    trk_off.close()
    trk, fps_on = run(True, frames)
    out["fps_off"], out["fps_on"] = fps_off, fps_on
    res, times = [], []
    while True:                        # one keyframe per call: each keyframe's own time (the call synchronises)
        t0 = time.perf_counter(); r = trk.detect_loops(capacity=1); dt = time.perf_counter() - t0
        if not r:
            break
        res += r; times.append(1e3 * dt)
    trk.close()
    out["keyframes"] = len(res)
    out["detect_ms_per_keyframe"] = float(np.mean(times)) if times else "not measured"
    stages = {}
    for r in res:
        stages[r["stage_name"]] = stages.get(r["stage_name"], 0) + 1
    out["stages"] = stages
    ver = [t for t, r in zip(times, res) if r["stage_name"] in ("loop", "fitness")]
    out["verify_ms"] = float(np.median(ver)) if ver else "not measured"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
