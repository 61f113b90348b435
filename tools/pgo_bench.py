"""Pose-graph optimisation on the GPU (kt_op_pgo_optimise): seeded drifted chains of 10^4 and 10^5 nodes with L = 1, 16, 64 loops.

Prints one JSON line: the GPU's name and power limit read in the same run, then per case (n nodes, L loops, it Gauss-Newton steps)
  solve_ms   one kt_op_pgo_optimise call, CUDA events around it, median of --reps (includes its allocations and uploads)
  step_ms    one Gauss-Newton step on the device (assembly to the chi2 of the updated poses), CUDA events inside the library
             (kt_pgo_report::step_ms, the mean over the steps of a call), median of --reps
  kernel_ms  per kernel, summed over one call, from a separate torch.profiler pass (names without the pgo_ / _kernel affixes)
  oracle_cpu_s  the scipy oracle on the same graph: a CPU figure, one run
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,100000")
    ap.add_argument("--loops", default="1,16,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200.binding import PGO_FACTOR_DTYPE
    from oracle import pgo_oracle as P
    if not torch.cuda.is_available():
        raise SystemExit("pgo_bench: no CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": smi.splitlines()[0] if smi else "unknown", "cases": []}
    for n in [int(s) for s in a.sizes.split(",")]:
        for L in [int(s) for s in a.loops.split(",")]:
            Xgt, Xd, loops = P.synthetic_chain(n + L, n, L)
            fi, fj, fz = P.chain_factors(Xd, loops)
            f = np.zeros(len(fi), PGO_FACTOR_DTYPE); f["i"] = fi; f["j"] = fj; f["z"] = fz
            poses = torch.from_numpy(np.ascontiguousarray(Xd)).cuda(); fd = torch.from_numpy(f.view(np.uint8)).cuda()
            res = torch.empty_like(poses)
            rep = kb.ops.pgo_optimise(poses, fd, res)                       # warm-up
            times, steps = [], []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); rep = kb.ops.pgo_optimise(poses, fd, res); e1.record(); torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1)); steps.append(rep.step_ms)
            case = {"n": n, "L": L, "it": rep.iterations, "solve_ms": round(float(np.median(times)), 2), "step_ms": round(float(np.median(steps)), 2)}
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                kb.ops.pgo_optimise(poses, fd, res); torch.cuda.synchronize()
            k = {}
            for ev in prof.key_averages():
                if "pgo_" in ev.key:
                    name = ev.key.split("pgo_")[1].split("(")[0].split("<")[0].replace("_kernel", "")
                    k[name] = round(k.get(name, 0.0) + ev.device_time_total / 1000.0, 2)
            case["kernel_ms"] = k
            if not a.no_oracle:
                t0 = time.perf_counter(); P.optimise(Xd, fi, fj, fz); case["oracle_cpu_s"] = round(time.perf_counter() - t0, 1)
            out["cases"].append(case)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
