#!/usr/bin/env python3
"""Cost of welding the map mesh on the GPU (kt_weld.cu: kt_op_weld_meshes; kt_get_map_mesh with weld).

Workload (seeded, tools-only):
  * a --vol^3 (default 1024^3) synthetic TSDF on the device: a sphere of radius 0.3 vol with a sinusoidal ripple, truncated at 4 voxels,
    every voxel observed with weight 20; cut along x into --slabs slabs that overlap by 3 planes (the tracker's overlap 2 plus the
    shared upper plane), each meshed with kt_op_mesh_volume_keyed on the device.  The weld of the concatenation is timed by its
    report's CUDA events (sort: keys and both radix sorts; weld: winners, representatives and the output; total: the whole call with
    its allocations and three host round trips), medians of --reps, and checked against kt_op_mesh_volume of the whole volume;
  * kt_get_map_mesh (which 0, weld 1) on a tracked map: --frames of the synthetic stream at 640 x 480 into 512^3 with slice meshing
    on; its report's upload / sort / weld / download / total device times and the host time of the call, medians of --reps.
Prints one JSON line with the GPU's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.map_bench import gpu_facts, med  # noqa: E402


def sdf_volume(V):
    import torch
    tsdf = torch.empty((V, V, V), dtype=torch.int16, device="cuda")
    color = torch.empty((V, V, V, 4), dtype=torch.uint8, device="cuda")
    ax = torch.arange(V, device="cuda", dtype=torch.float32)
    y, x = torch.meshgrid(ax, ax, indexing="ij")
    for z in range(0, V, 64):
        zz = ax[z:z + 64].view(-1, 1, 1)
        d = torch.sqrt((x - 0.48 * V) ** 2 + (y - 0.51 * V) ** 2 + (zz - 0.5 * V) ** 2) - 0.3 * V + 2.0 * torch.sin(x * 0.05) * torch.cos(y * 0.04)
        tsdf[z:z + 64] = torch.trunc(torch.clamp(d / 4.0, -1.0, 1.0) * 32767).to(torch.int16)
        col = torch.stack([(x * 0.25).to(torch.uint8).expand_as(d), (y * 0.25).to(torch.uint8).expand_as(d), (zz * 0.25).to(torch.uint8).expand_as(d),
                           torch.full_like(d, 20, dtype=torch.uint8)], -1)
        color[z:z + 64] = col
    return tsdf, color


def slab_weld(kb, V, slabs, reps):
    import torch
    tsdf, color = sdf_volume(V)
    size = [6.0 * V / 512] * 3
    cuts = [round(V * i / slabs) for i in range(slabs + 1)]
    boxes = [(max(cuts[i] - 2, 0), min(cuts[i + 1] + 1, V), 0, V, 0, V) for i in range(slabs)]
    parts = []
    for b in boxes:
        st, nv, nt = kb.ops.mesh_volume_keyed_into(tsdf, color, V, size, (0, 0, 0), (0, 0, 0), b, 8, None, None, 0, None, None, 0)
        v = torch.empty(max(nv, 1) * 32, dtype=torch.uint8, device="cuda"); e = torch.empty(max(nv, 1) * 4, dtype=torch.int32, device="cuda")
        t = torch.empty(max(nt, 1) * 3, dtype=torch.int32, device="cuda"); k = torch.empty(max(nt, 1) * 4, dtype=torch.int32, device="cuda")
        st, nv, nt = kb.ops.mesh_volume_keyed_into(tsdf, color, V, size, (0, 0, 0), (0, 0, 0), b, 8, v, e, nv, t, k, nt)
        kb.binding._check(st)
        parts.append((v[:nv * 32], e[:nv * 4], t[:nt * 3], k[:nt * 4], nv, nt))
    vo = np.concatenate([[0], np.cumsum([p[4] for p in parts])]); to = np.concatenate([[0], np.cumsum([p[5] for p in parts])])
    dv = torch.cat([p[0] for p in parts]); de = torch.cat([p[1] for p in parts]); dt = torch.cat([p[2] for p in parts]); dk = torch.cat([p[3] for p in parts])
    ov = torch.empty(int(vo[-1]) * 32, dtype=torch.uint8, device="cuda"); ot = torch.empty(int(to[-1]) * 12, dtype=torch.uint8, device="cuda")
    reports = []
    for r in range(reps + 1):                                           # the first call warms up CUB and the allocator
        st, nv, nt, rep = kb.ops.weld_meshes_into(dv, de, vo, dt, dk, to, ov, int(vo[-1]), ot, int(to[-1]))
        kb.binding._check(st)
        if r:
            reports.append(rep)
    whole = kb.ops.mesh_volume(tsdf, color, V, size, (0, 0, 0), (0, 0, 0), (0, V, 0, V, 0, V), 8)
    same = ov[:nv * 32].cpu().numpy().tobytes() == whole[0].tobytes() and np.array_equal(ot[:nt * 12].cpu().numpy().view(np.uint32).reshape(-1, 3), whole[1])
    rep = reports[-1]
    total = med([q["total_ms"] for q in reports])
    return dict(vol=V, slabs=slabs, input_tris=rep["input_tris"], output_tris=rep["output_tris"], input_verts=rep["input_verts"],
                output_verts=rep["output_verts"], repeated_cells=rep["repeated_cells"], equals_whole_volume_mesh=bool(same),
                sort_ms=med([q["sort_ms"] for q in reports]), weld_ms=med([q["weld_ms"] for q in reports]), total_ms=total,
                input_tris_per_s=round(rep["input_tris"] / (total * 1e-3), 1))


def tracker_export(kb, frames, reps):
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=480, cols=640, vol=512, odometry=0))
    trk.set_slice_meshing(True, 8)
    for k in range(frames):
        d, c = synth.render(k, 640, 480)
        trk.process_frame(d, c, k)
    trk.finalise()
    nv = C.c_size_t(0); nt = C.c_size_t(0); rep = kb.binding.WeldReport()
    kb.binding._check(trk.lib.kt_get_map_mesh(trk.h, 0, 1, None, C.c_size_t(0), None, C.c_size_t(0), C.byref(nv), C.byref(nt), C.byref(rep)))
    v = np.zeros(nv.value, kb.binding.MESH_VERTEX_DTYPE); t = np.zeros((nt.value, 3), np.uint32)
    reports, host = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        kb.binding._check(trk.lib.kt_get_map_mesh(trk.h, 0, 1, kb.binding._ptr(v), C.c_size_t(len(v)), kb.binding._ptr(t), C.c_size_t(len(t)),
                                                  C.byref(nv), C.byref(nt), C.byref(rep)))
        host.append((time.perf_counter() - t0) * 1e3)
        reports.append(rep.as_dict())
    r = reports[-1]
    out = dict(frames=frames, slices=r["meshes"], input_tris=r["input_tris"], output_tris=r["output_tris"], input_verts=r["input_verts"],
               output_verts=r["output_verts"], repeated_cells=r["repeated_cells"], host_ms=med(host))
    for key in ("upload_ms", "sort_ms", "weld_ms", "download_ms", "total_ms"):
        out[key] = med([q[key] for q in reports])
    trk.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--vol", type=int, default=1024)
    ap.add_argument("--slabs", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--frames", type=int, default=72)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import kintinuous_b200 as kb
    if not kb.cuda_available():
        raise SystemExit("weld_bench: no CUDA device (there is no CPU path)")
    res = dict(gpu_facts())
    res["slab_weld"] = [slab_weld(kb, a.vol, n, a.reps) for n in a.slabs]
    res["tracker_map_mesh"] = tracker_export(kb, a.frames, a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
