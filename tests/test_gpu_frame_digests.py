"""The whole-frame odometry kernels against digests of their results recorded on an H100.

icp_frame_kernel and rgbd_frame_kernel reduce each warp's 29 running sums with a fixed shuffle tree (warp_transpose_sum, kt_frame.cuh)
and then sum exactly over the grid, so a change to how the tree is compiled or scheduled must not change a bit.  Over the synthetic
stream the poses, the per-iteration normal equations (trace) and the current and model maps of every level must hash to the recorded
values: ICP-only at 640x480 (every level fully staged in shared memory) and 1280x960 (level 0 partly streamed from global memory), each
also with a two-pass stage (KT_ICP_STAGE_PASSES=2), and ICP + RGB-D at 640x480.

The digests were recorded on an H100 SXM (132 SMs).  The pixel partition over CTAs, and so the float partials, follow the SM count,
so on another part the test only checks that the stage sizes agree with each other."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

GOLDEN_SMS = 132
GOLDEN = {"icp 640x480": "ce2d1d9a7a77acf609b853927c40376f67500e3408b05ac6acc9ef968a0cc76e",
          "icp 1280x960": "19323f33e90c4fd578b14269cb0438b89ad2ab9cdbd53fbe94f358ba12996594",
          "icp+rgbd 640x480": "c85cd0cd860bbe20c1fee6919a78ad4e1fec80a754f8abb846864b6e6b828f1b"}

SCRIPT = r"""
import hashlib, json
import numpy as np
import kintinuous_b200 as kb
from kintinuous_b200 import synth
out = {}
for name, odometry, rows, cols, n in (("icp", 0, 480, 640, 8), ("icp", 0, 960, 1280, 4), ("icp+rgbd", 2, 480, 640, 8)):
    trk = kb.Tracker(kb.Config.default(rows=rows, cols=cols, vol=256, odometry=odometry))
    h = hashlib.sha256()
    for k in range(n):
        d, c = synth.render(k, cols, rows)
        p = trk.process_frame(d, c, k)
        R, t, gc, w = p.as_tuple()
        h.update(np.ascontiguousarray(R).tobytes()); h.update(np.ascontiguousarray(t).tobytes())
        h.update(trk.trace().tobytes())
    for lvl in range(3):
        for which in range(4):
            h.update(np.ascontiguousarray(trk.download_map(which, lvl)).tobytes())
    out[f"{name} {cols}x{rows}"] = h.hexdigest()
    trk.close()
print("DIGEST", json.dumps(out))
"""


def _digests(extra_env):
    from conftest import ROOT
    env = dict(os.environ, PYTHONPATH=ROOT, **extra_env)
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads([l for l in r.stdout.splitlines() if l.startswith("DIGEST")][0][len("DIGEST "):])


def test_frame_kernels_match_recorded_digests(built):
    import torch
    default = _digests({})
    stage2 = _digests({"KT_ICP_STAGE_PASSES": "2"})
    assert default == stage2, (default, stage2)
    if torch.cuda.get_device_properties(0).multi_processor_count == GOLDEN_SMS:
        assert default == GOLDEN, default
