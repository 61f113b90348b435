"""A refused device allocation fails only the call that asked for it.  cudaMalloc records a failure as the runtime's last error; the
library clears it (kt_mem.hpp), so the next launch check of a later frame does not report it as a failed launch."""
import pytest

pytestmark = pytest.mark.gpu

ROWS, COLS, V, FRAMES = 240, 320, 256, 60


def _track(kb, act=None, n=FRAMES):
    from kintinuous_b200 import synth
    trk = kb.Tracker(kb.Config.default(rows=ROWS, cols=COLS, vol=V, odometry=0, voxel_shift=2))
    trk.set_slice_processing(True, 8)
    poses, traces = [], []
    for k in range(n):
        if act is not None and k == n // 2:
            act(trk)
        d, c = synth.render(k, COLS, ROWS)
        poses.append(bytes(trk.process_frame(d, c, k)))
        traces.append(trk.trace().tobytes())
    trk.finalise()
    return trk, poses, traces


def test_refused_loop_store_leaves_tracking_intact(built):
    import kintinuous_b200 as kb
    _, ref_poses, ref_traces = _track(kb)

    def act(trk):
        # 2^20 keyframes of 2^20 features: the depth store alone is 2^20 * 320 * 240 * 2 B = 161 GB, twice the card's memory, so the
        # store is refused whatever order its arrays are allocated in, before any kernel sees them
        with pytest.raises(kb.KtError, match="error -2"):
            trk.set_loop_detection(max_keyframes=1 << 20, max_features=1 << 20)
        assert trk.num_keyframes() == (0, False)

    trk, poses, traces = _track(kb, act)
    assert poses == ref_poses and traces == ref_traces
    assert trk.num_keyframes() == (0, False)
    trk.set_loop_detection()
