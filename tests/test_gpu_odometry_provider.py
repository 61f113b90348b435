"""The OdometryProvider entry points of the C ABI (kt_odometry_first_run / kt_odometry_increment) against the tracker: a context that is
given the tracker's previous pose and predicted maps, and the same depth / colour frame, must estimate the tracker's pose bit for bit.
The tracker does not shift its volume here, so the pose it reports is the odometry's estimate itself."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROWS, COLS, VOL, FRAMES, LEVELS = 240, 320, 128, 6, 4


def _pyramid(trk, which):
    """Device copies of one map of the tracker at every level, and the host array of their pointers the C ABI takes."""
    import torch
    maps = [torch.from_numpy(trk.download_map(which, l)).cuda() for l in range(LEVELS)]
    torch.cuda.synchronize()           # the library's streams do not wait for torch's
    return maps, (C.c_void_p * LEVELS)(*[m.data_ptr() for m in maps])


@pytest.mark.parametrize("odometry", [0, 1, 2])
def test_odometry_provider_matches_the_tracker(built, odometry):
    import torch
    import kintinuous_b200 as kb
    from kintinuous_b200 import synth
    from kintinuous_b200 import binding
    from kintinuous_b200.binding import _check, _ptr
    lib = binding.load()
    cfg = kb.Config.default(rows=ROWS, cols=COLS, vol=VOL, odometry=odometry, parked=1)
    trk = kb.Tracker(cfg)
    odo = kb.Tracker(cfg)              # only its context is used: the odometry's scratch and the photometric pyramids between calls
    frames = [synth.render(k, COLS, ROWS) for k in range(FRAMES)]
    dev = [(torch.from_numpy(d.view(np.int16)).cuda(), torch.from_numpy(c).cuda()) for d, c in frames]
    torch.cuda.synchronize()
    trk.process_frame(frames[0][0], frames[0][1], 0)
    _check(lib.kt_odometry_first_run(odo.h, _ptr(dev[0][0]), _ptr(dev[0][1])))
    for k in range(1, FRAMES):
        prev = trk.pose()
        Rprev = np.array(prev.R, np.float32); tprev = np.array(prev.t, np.float32)
        vg, vgp = _pyramid(trk, 2)
        ng, ngp = _pyramid(trk, 3)
        p = trk.process_frame(frames[k][0], frames[k][1], k)
        want_R = np.array(p.R, np.float32); want_t = np.array(p.t, np.float32)
        calls = []
        if odometry == 0:
            vc, vcp = _pyramid(trk, 0)      # the caller's current maps: the frame itself is not needed
            nc, ncp = _pyramid(trk, 1)
            calls.append((None, None, vcp, ncp))
        calls.append((dev[k][0], dev[k][1], None, None))
        for depth, rgb, vcurr, ncurr in calls:
            R = np.zeros(9, np.float32); t = np.zeros(3, np.float32)
            _check(lib.kt_odometry_increment(odo.h, _ptr(depth), _ptr(rgb), _ptr(Rprev), _ptr(tprev), vgp, ngp, vcurr, ncurr, _ptr(R), _ptr(t)))
            assert R.tobytes() == want_R.tobytes() and t.tobytes() == want_t.tobytes(), (k, vcurr is not None, R, want_R, t, want_t)
        assert np.abs(want_t - tprev).max() > 0, k          # the camera moves: the comparison is not of two copies of tprev
    odo.close(); trk.close()
