"""The volume operators -- integrate, ray cast, extract, clear -- from every side of the cube and at sides that are not powers of two,
against what the reference's own CUDA operators computed over the same table of views (tests/volume_views.py; fixtures
tests/golden/ref_views_*.npz, recorded by tools/make_golden.py).

Bar, as for the other operator parity tests: 0 LSB for TSDF, weights and colours (every voxel, by digest), bit-identical vertex, normal
and colour maps, identical multisets of extracted points, and identical cleared volumes.  (A slab whose extraction by the reference is
not well defined -- it loses or misplaces points that other warps append after it published its count, DESIGN.md R1 -- is not recorded,
and so not compared.)  Each view must also show something: a minimum
of touched voxels and ray hits -- except the camera that looks away from the cube, which must touch and hit nothing."""
import os
import subprocess
import sys

import numpy as np
import pytest

import volume_views as vv
from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

CASES = [(V, vs, n) for V, vs, names in vv.table() for n in names]


def _fixture(V, vs):
    return np.load(os.path.join(GOLDEN, f"ref_views_{vv.case_key(V, vs)}.npz"))


def _where(got, want, name, bad):
    """A readable account of the first mismatches: which output, and for voxels / pixels, where."""
    msg = []
    for k in bad[:6]:
        what = k.split(".", 1)[1]
        if what == "tsdf" or what == "color":
            idx = want[f"{name}.vox_idx"]
            t = np.flatnonzero(got[f"{name}.vox_tsdf"] != want[f"{name}.vox_tsdf"]) if got[f"{name}.vox_tsdf"].shape == want[f"{name}.vox_tsdf"].shape else []
            msg.append(f"{k}: sampled voxels differing in TSDF {[int(idx[i]) for i in t[:5]]}")
        elif what.endswith("_v") and what.startswith("ray"):
            tag = what[:-2]
            msg.append(f"{k}: hits {got.get(f'{name}.{tag}_hits')} vs {int(want[f'{name}.{tag}_hits'])}")
        elif what.startswith("ext_") and not what.endswith("_n"):
            msg.append(f"{k}: {got.get(f'{name}.{what}_n')} vs {int(want[f'{name}.{what}_n'])} points")
        else:
            msg.append(k)
    return "; ".join(msg)


@pytest.mark.parametrize("V,vs,name", CASES, ids=[f"{vv.case_key(V, vs)}-{n}" for V, vs, n in CASES])
def test_view_vs_reference(built, V, vs, name):
    import torch
    import kintinuous_b200 as kb
    want = _fixture(V, vs)
    R, t, wrap = [(R, t, w) for n, R, t, w in vv.views(V, vs) if n == name][0]
    got = {f"{name}.{k}": v for k, v in vv.run_view(kb.ops, torch, V, vs, name, R, t, wrap).items()}
    # not vacuous: the view integrates a surface and sees it; the camera facing away touches and hits nothing
    touched, hits = int(want[f"{name}.touched"]), int(want[f"{name}.ray0_hits"])
    if name == "look_away":
        assert touched == 0 and hits == 0 and int(want[f"{name}.ray1_hits"]) == 0, (touched, hits)
    else:
        assert touched >= 5000 and hits >= 1000, (touched, hits)
    bad = vv.compare(got, want, f"{name}.")
    assert not bad, f"{vv.case_key(V, vs)} {name}: {_where(got, want, name, bad)}"


@pytest.mark.parametrize("V", vv.VOLS)
def test_cleared_planes_vs_reference(built, V):
    """Runs of planes along every axis, forward and back, across the end of storage, on a sentinel-filled volume: the same storage planes
    zeroed, each whole.  (At 200 the x runs are absent: the reference's clearVolumeX leaves the volume unless V % 16 == 0.)"""
    import torch
    import kintinuous_b200 as kb
    want = _fixture(V, (vv.SIZE,) * 3)
    got = {f"clear.{k}": v for k, v in vv.cleared_planes(kb.ops, torch, V).items()}
    assert sorted(got) == sorted(k for k in want.files if k.startswith("clear."))
    assert not vv.compare(got, want, "clear."), vv.compare(got, want, "clear.")


_VARIANT_SCRIPT = r"""
import os, sys
sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import numpy as np
import torch
import kintinuous_b200 as kb
import volume_views as vv
V = int(sys.argv[1])
want = np.load(os.path.join("tests", "golden", f"ref_views_{V}.npz"))
got = vv.run_case(kb.ops, torch, V, (vv.SIZE,) * 3)
bad = vv.compare(got, want)
print("VIEWS", len([k for k in want.files if k.endswith(".touched")]), "MISMATCH", bad[:20])
"""


@pytest.mark.parametrize("variant", [{"KT_FORCE_IDX64": "1"}, {"KT_INT_NOBOX": "1"}], ids=["idx64", "nobox"])
def test_384_table_under_kernel_variants(built, variant):
    """The 384 table through two instances the default configuration does not take at that size: 64-bit voxel indices
    (raycast_kernel<false, size_t> and the 64-bit integrate), and integrate launched over the whole volume instead of the frustum's box
    of storage tiles.  Both must reproduce the reference's outputs view by view -- the culls are exact, not just close."""
    env = dict(os.environ, PYTHONPATH=ROOT, **variant)
    r = subprocess.run([sys.executable, "-c", _VARIANT_SCRIPT, "384"], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("VIEWS")][0]
    assert line.endswith("MISMATCH []") and int(line.split()[1]) == len(vv.views(384)), line
