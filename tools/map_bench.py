#!/usr/bin/env python3
"""Cost of the whole-map export on the GPU (kt_map.cu: kt_op_voxel_grid; kt_get_map_cloud).

Workload (seeded, tools-only): --sizes clouds of 48-byte kt_point_xyzrgbnormal records (default 10^7 and 5 x 10^7), uniformly random in a
box of 0.4 points per leaf at the default voxel edge (6 m / 512), so an occupied leaf holds 1.2 points on average -- about the share of
points a map's overlap planes repeat.  Per size, device times (CUDA events, median of --reps):
  * upload: the records from pinned host memory to the device (H2D);
  * voxel_grid: the whole kt_op_voxel_grid call (bounds, keys, sort, leaf starts, centroids, two host round trips, its allocations);
  * download: the filtered cloud back to pinned memory (D2H);
  * sort / centroids: per-kernel device time from a separate torch.profiler pass -- keys + CUB radix sort, and head flags + CUB scan +
    leaf starts + centroid kernel.
Then kt_get_map_cloud (which 0, dedupe 1) on a tracked map (--frames of the synthetic stream at 640 x 480 into 512^3 with slice
processing on): its report's upload / sort / centroid / download / total device times and the host time of the call, medians.
Prints one JSON line with the GPU's name and power limit, read in the same run."""
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, smmax = [s.strip() for s in out.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock_max=smmax)
    except Exception as e:
        return dict(gpu="not read: %s" % e)


def med(v):
    return round(float(np.median(v)), 3)


def cloud(torch, n, leaf, seed):
    """n records on the device (float32 [n, 12] = x y z 1 nx ny nz 0 rgba curvature 0 0)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    side = (n / 0.4) ** (1.0 / 3.0) * leaf
    r = torch.zeros((n, 12), dtype=torch.float32, device="cuda")
    r[:, 0:3] = torch.rand((n, 3), generator=g, device="cuda") * side - side / 2
    r[:, 3] = 1.0
    nrm = torch.randn((n, 3), generator=g, device="cuda")
    r[:, 4:7] = nrm / nrm.norm(dim=1, keepdim=True)
    r[:, 8] = torch.randint(0, 1 << 24, (n,), generator=g, device="cuda", dtype=torch.int32).view(torch.float32)
    r[:, 9] = torch.rand((n,), generator=g, device="cuda") * 0.3
    return r


def bench_operator(torch, kb, n, leaf, reps):
    dev = cloud(torch, n, leaf, 7)
    host = torch.empty(dev.shape, dtype=dev.dtype, pin_memory=True)
    host.copy_(dev)
    out = torch.empty_like(dev)
    back = torch.empty(dev.shape, dtype=dev.dtype, pin_memory=True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    t = {"upload": [], "voxel_grid": [], "download": []}
    m = skip = 0
    for rep in range(reps + 1):
        ev[0].record()
        dev.copy_(host, non_blocking=True)
        ev[1].record()
        m, skip = kb.ops.voxel_grid(dev, n, 1, leaf, out, n)
        ev[2].record()
        back[:m].copy_(out[:m], non_blocking=True)
        ev[3].record()
        torch.cuda.synchronize()
        if rep:                                                      # the first round loads the modules
            t["upload"].append(ev[0].elapsed_time(ev[1])); t["voxel_grid"].append(ev[1].elapsed_time(ev[2]))
            t["download"].append(ev[2].elapsed_time(ev[3]))
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        kb.ops.voxel_grid(dev, n, 1, leaf, out, n)
        torch.cuda.synchronize()
    cat = {"bounds": 0.0, "sort": 0.0, "centroids": 0.0, "other": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if not us:
            continue
        k = e.key
        if "map_bounds" in k:
            cat["bounds"] += us
        elif "map_keys" in k or "Radix" in k or "Onesweep" in k or "radix" in k:
            cat["sort"] += us
        elif "map_heads" in k or "map_starts" in k or "map_centroid" in k or "Scan" in k:
            cat["centroids"] += us
        else:
            cat["other"] += us
    r = {k: med(v) for k, v in t.items()}
    r.update({f"{k}_kernels_ms": round(v / 1000.0, 3) for k, v in cat.items()})
    r.update(points=n, leaves=int(m), pcl_would_skip=int(skip),
             pipeline_ms=round(r["upload"] + r["voxel_grid"] + r["download"], 3))
    del dev, host, out, back
    torch.cuda.empty_cache()
    return r


def bench_tracker(torch, kb, frames, reps):
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=480, cols=640, vol=512, odometry=0, voxel_shift=2))
    trk.set_slice_processing(True, 8)
    for k in range(frames):
        d, c = synth.render(k, 640, 480)
        trk.process_frame(d, c, k)
    trk.finalise()
    import ctypes as C
    n = C.c_size_t(0)
    from kintinuous_b200.binding import MapReport, POINT_NORMAL_DTYPE
    rep = MapReport()
    assert trk.lib.kt_get_map_cloud(trk.h, 0, 1, None, C.c_size_t(0), C.byref(n), C.byref(rep)) == 0
    out = np.zeros(n.value, POINT_NORMAL_DTYPE)
    rows = []
    for _ in range(reps):
        t0 = time.perf_counter()
        assert trk.lib.kt_get_map_cloud(trk.h, 0, 1, out.ctypes.data_as(C.c_void_p), C.c_size_t(len(out)), C.byref(n), C.byref(rep)) == 0
        rows.append(dict(rep.as_dict(), host_ms=(time.perf_counter() - t0) * 1000.0))
    t0 = time.perf_counter()
    trk.map_cloud(0, False)
    copy_ms = (time.perf_counter() - t0) * 1000.0
    r = {k: (med([x[k] for x in rows]) if isinstance(rows[0][k], float) else rows[0][k]) for k in rows[0]}
    r.update(frames=frames, slices=trk.num_slices(), concat_host_copy_ms=round(copy_ms, 3))
    trk.close()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000000,50000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=300)
    a = ap.parse_args()
    import torch
    import kintinuous_b200 as kb
    if not torch.cuda.is_available():
        sys.exit("map_bench: needs a CUDA device")
    leaf = float(np.float32(6.0 / 512))
    res = dict(gpu_facts(), leaf=leaf, reps=a.reps)
    res["operator"] = [bench_operator(torch, kb, int(s), leaf, a.reps) for s in a.sizes.split(",")]
    res["kt_get_map_cloud"] = bench_tracker(torch, kb, a.frames, a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
