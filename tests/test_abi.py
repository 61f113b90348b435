"""The C-ABI library loads without a GPU, exports every symbol include/kintinuous_b200.h declares, and fails loudly
(no CPU fallback) when asked to compute without a CUDA device."""
import ctypes
import os
import re

import numpy as np
import pytest

from conftest import ROOT


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "kintinuous_b200.h")).read()
    return sorted(set(re.findall(r"KT_API\s+[\w\s\*]+?\b(kt_[a-z0-9_]+)\s*\(", hdr)))


def test_header_declares_the_boundary():
    syms = declared_symbols()
    assert len(syms) >= 40
    for must in ("kt_create", "kt_process_frame", "kt_process_frame_device", "kt_finalise", "kt_volume_export_reference_layout",
                 "kt_op_icp_step", "kt_op_integrate", "kt_op_raycast", "kt_op_extract_slice", "kt_op_rgb_step", "kt_op_rgb_residual"):
        assert must in syms


def test_library_exports_every_declared_symbol(built):
    import kintinuous_b200 as kb
    lib = ctypes.CDLL(kb.lib_path())
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, missing


def test_every_entry_point_cites_the_reference():
    hdr = open(os.path.join(ROOT, "include", "kintinuous_b200.h")).read()
    # every operator names the reference function / file it replaces
    for name in ("bilateralFilter", "pyrDown", "createVMap", "createNMap", "tranformMaps", "resizeVMap", "icpStep", "integrateTsdfVolume",
                 "raycast", "extractCloudSlice", "clearVolume", "initVolume", "KintinuousTracker::processFrame", "reduce.cu", "tsdf_volume.cu"):
        assert name in hdr, name


def test_no_cpu_fallback(built):
    import kintinuous_b200 as kb
    if kb.cuda_available():
        pytest.skip("a GPU is present")
    with pytest.raises(kb.KtError):
        kb.Tracker(kb.Config.default(vol=128))
    a = np.zeros((8, 32), np.uint16)
    with pytest.raises(kb.KtError):
        kb.ops.bilateral(a, a.copy(), 8, 32)


def test_config_validation(built):
    import kintinuous_b200 as kb
    lib = kb.load()
    h = ctypes.c_void_p()
    bad = kb.Config.default(vol=100)
    assert lib.kt_create(ctypes.byref(bad), ctypes.byref(h)) != 0
    assert b"vol" in lib.kt_last_error() or b"CUDA" in lib.kt_last_error()
    assert lib.kt_create(None, ctypes.byref(h)) != 0


@pytest.mark.parametrize("vol", [100, 33, 4, 0, -8])
def test_volume_operators_refuse_a_side_that_is_not_a_multiple_of_8(built, vol):
    """Every volume operator refuses vol % 8 != 0 (and vol <= 0) with KT_ERR_INVALID before it launches anything: at V = 100 the y / z
    clear's 16-byte row stores would be misaligned and miss each row's last 4 voxels, at V = 33 init_volume would leave the last voxel
    unwritten.  The pointers are NULL: a call that got past the check would fail differently (or fault), so this needs no GPU."""
    import kintinuous_b200 as kb
    ops = kb.ops
    eye, t3, intr, vs = np.eye(3, dtype=np.float32), np.full(3, 3.0, np.float32), np.array([132.0, 132.0, 80.0, 66.75], np.float32), [6.0] * 3
    calls = {
        "kt_op_init_volume": lambda: ops.init_volume(None, None, vol),
        "kt_op_clear_volume": lambda: ops.clear_volume(1, 0, None, None, vol, 0, 14),
        "kt_op_integrate": lambda: ops.integrate(None, 120, 160, intr, vs, eye, t3, 0.06, None, None, vol, (0, 0, 0), None, None, 1, None),
        "kt_op_raycast": lambda: ops.raycast(intr, eye, t3, 0.06, vs, None, vol, None, None, 120, 160, (0, 0, 0), None, None),
        "kt_op_extract_slice": lambda: ops.extract_slice(None, vs, vol, None, 10, (0, 0, 0), None, (0, 8, 0, 8, 0, 8), 1, (0, 0, 0)),
        "kt_op_mesh_volume": lambda: ops.mesh_volume_into(None, None, vol, vs, (0, 0, 0), (0, 0, 0), (0, 8, 0, 8, 0, 8), 8, None, 0, None, 0),
        "kt_op_mesh_volume_keyed": lambda: ops.mesh_volume_keyed_into(None, None, vol, vs, (0, 0, 0), (0, 0, 0), (0, 8, 0, 8, 0, 8), 8, None, None, 0,
                                                                     None, None, 0),
    }
    for name, call in calls.items():
        with pytest.raises(kb.KtError) as e:
            call()
        assert f"{name}: vol {vol} is not a positive multiple of 8" in str(e.value), (name, str(e.value))


def test_product_never_touches_the_oracle():
    """The product path must not import, link or execute anything under oracle/."""
    pkg = os.path.join(ROOT, "kintinuous_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", "Makefile")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle/" not in txt.replace("the oracle/", "") or f == "__init__.py", (dirpath, f)
                assert "import oracle" not in txt and "from oracle" not in txt, (dirpath, f)
                assert "kt_oracle" not in txt and "refbind" not in txt and "libkt_ref" not in txt, (dirpath, f)
