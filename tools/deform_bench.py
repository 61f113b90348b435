#!/usr/bin/env python3
"""Cost of map deformation on the GPU (kt_deform.cu) on a loop-closure-sized workload, through the kt_op_deform_* operators.

Workload (seeded, tools-only): a 10-minute trajectory at 30 Hz (18 000 dense poses, one pose constraint each), nodes every 0.8 m (the
reference's -dg default; about 1000 nodes), 5 M map vertices as 48-byte kt_point_xyzrgbnormal records, a time-varying correction
(rotation about +y up to 20 degrees and a translation up to 6.7 m, large enough to pass the reference's constraint-error early-out at
this many constraints).  Prints one JSON line with
  * device times (CUDA events, median of --reps) of: map upload (H2D) and download (D2H) from / to pinned memory, vertex weights,
    the whole Gauss-Newton optimisation (its iterations and its time per iteration), apply;
  * per-kernel device time from a separate torch.profiler pass: residual, assembly, factor + solve, weights, apply, per launch;
  * apply's bytes (48 in + 48 out + 16 ids + 32 weights per vertex) over its time, and over the H100 SXM data-sheet 3.35 TB/s;
  * the GPU's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--poses", type=int, default=18000)
    ap.add_argument("--verts", type=int, default=5_000_000)
    ap.add_argument("--spacing", type=float, default=0.8)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200.binding import POINT_NORMAL_DTYPE
    from oracle import deform_oracle as D
    if not torch.cuda.is_available():
        sys.exit("deform_bench: needs a CUDA device")
    step = a.spacing * 1000 / a.poses
    times, pos, vt, v, nrm = D.synthetic(11, a.poses, a.verts, step=step, radius=60.0, spread=2.0)
    o = np.argsort(vt, kind="stable")                                     # a map is stored slice by slice, i.e. in time order
    vt, v, nrm = vt[o], v[o], nrm[o]
    take = D.sample_nodes(pos, a.spacing)
    tf = (times - times[0]) / float(times[-1] - times[0])
    WR, Wt = D.warp(tf, 20.0, (5.0, -2.0, 4.0))
    corr = np.einsum("nij,nj->ni", WR, pos.astype(np.float64)) + Wt
    recs = np.zeros(a.verts, POINT_NORMAL_DTYPE)
    for i, c in enumerate("xyz"):
        recs[c] = v[:, i]; recs["n" + c] = nrm[:, i]
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).cuda()
    n = len(take); m = a.poses; N = a.verts
    npos = dev(pos[take]).view(torch.float32).view(n, 3); nt = dev(times[take])
    cs = dev(pos); ct = dev(times).view(torch.int64); cd = dev(corr)
    cids = torch.empty(m * 16, dtype=torch.uint8, device="cuda"); cw = torch.empty(m * 32, dtype=torch.uint8, device="cuda")
    params = torch.empty(n * 12, dtype=torch.float64, device="cuda")
    host_in = torch.from_numpy(recs.view(np.uint8)).pin_memory(); host_out = torch.empty_like(host_in).pin_memory()
    vth = torch.from_numpy(vt.view(np.int64)).pin_memory()
    pin = torch.empty(N * 48, dtype=torch.uint8, device="cuda"); pout = torch.empty_like(pin)
    vtd = torch.empty(N, dtype=torch.int64, device="cuda")
    ids = torch.empty(N * 16, dtype=torch.uint8, device="cuda"); w = torch.empty(N * 32, dtype=torch.uint8, device="cuda")

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); r = fn(); e1.record(); e1.synchronize()
        return e0.elapsed_time(e1), r

    phases = {k: [] for k in ("h2d", "weights", "optimise", "apply", "d2h")}
    rep = None
    for it in range(a.reps + 1):
        t = {}
        t["h2d"], _ = timed(lambda: (pin.copy_(host_in, non_blocking=True), vtd.copy_(vth, non_blocking=True)))
        kb.ops.deform_weights(npos, nt, cs, 2, ct, cids, cw)
        t["optimise"], rep = timed(lambda: kb.ops.deform_optimise(npos, cs.view(torch.float32).view(m, 3), cd, cids, cw, params))
        t["weights"], _ = timed(lambda: kb.ops.deform_weights(npos, nt, pin, 0, vtd, ids, w))
        t["apply"], _ = timed(lambda: kb.ops.deform_apply(npos, params, ids, w, pin, pout, 0, N))
        t["d2h"], _ = timed(lambda: host_out.copy_(pout, non_blocking=True))
        if it:                                                            # the first pass warms every shape up
            for k in phases:
                phases[k].append(t[k])
    med = {k + "_ms": float(np.median(v)) for k, v in phases.items()}
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        kb.ops.deform_optimise(npos, cs.view(torch.float32).view(m, 3), cd, cids, cw, params)
        kb.ops.deform_weights(npos, nt, pin, 0, vtd, ids, w)
        kb.ops.deform_apply(npos, params, ids, w, pin, pout, 0, N)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for key in ("deform_residual_kernel", "deform_assemble_kernel", "deform_solve_kernel", "deform_weight_kernel",
                    "deform_node_table_kernel", "deform_apply_kernel"):
            if key in e.key:
                kern[key] = dict(calls=e.count, avg_ms=e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3)
    out = host_out.numpy().view(POINT_NORMAL_DTYPE)
    assert np.isfinite(out["x"]).all() and rep.deformed == 1
    apply_bytes = N * (48 + 48 + 16 + 32)
    ak = kern.get("deform_apply_kernel", {}).get("avg_ms")
    res = dict(bench="deform", nodes=n, constraints=m, vertices=N, report=rep.as_dict(), **med,
               optimise_ms_per_iteration=med["optimise_ms"] / max(rep.iterations, 1), kernels=kern,
               apply_bytes=apply_bytes, apply_tb_s=apply_bytes / (med["apply_ms"] * 1e-3) / 1e12,
               apply_share_of_3_35_tb_s=apply_bytes / (med["apply_ms"] * 1e-3) / 3.35e12,
               apply_kernel_share_of_3_35_tb_s=(apply_bytes / (ak * 1e-3) / 3.35e12) if ak else None, **gpu_facts())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
