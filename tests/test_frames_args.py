"""Argument checks of the frame entry points (yb_network_predict_frames_u8, yb_network_detect_frames,
yb_network_submit_frames_u8): every invalid argument is rejected before any device work, so these run without a GPU,
and the Python mirror rejects frames of the wrong dtype, rank or channel count."""
import ctypes as C

import numpy as np
import pytest

import ybtest_util as util


@pytest.fixture(scope="module")
def net(tmp_path_factory):
    import yolo2_light_b200 as yb
    cfg, wts = util.model_files("tiny64", str(tmp_path_factory.mktemp("frames_args")))
    return yb.load_network(cfg, wts, batch=2)


def _call(net, which, frames, w, h, nimg, max_rows=64):
    """The raw C call; frames / w / h: Python lists or None (a null array)."""
    from yolo2_light_b200 import api
    L = api.lib()
    fa = None if frames is None else (C.c_void_p * max(len(frames), 1))(*frames)
    wa = None if w is None else (C.c_int * max(len(w), 1))(*w)
    ha = None if h is None else (C.c_int * max(len(h), 1))(*h)
    if which == "predict":
        ok = bool(L.yb_network_predict_frames_u8(net._h, fa, wa, ha, nimg, 0))
    elif which == "submit":
        ok = L.yb_network_submit_frames_u8(net._h, fa, wa, ha, nimg, 0, 0.5, 0.45, 1, 0, max_rows) >= 0
    else:
        rows = np.zeros((net.batch, max(max_rows, 1), 64), np.float32)
        counts = np.zeros(net.batch, np.int32)
        ok = L.yb_network_detect_frames(net._h, 0, wa, ha, nimg, 0.5, 0.45, 1, 0, rows.ctypes.data_as(C.c_void_p), max_rows,
                                        counts.ctypes.data_as(C.c_void_p)) >= 0
    api._check(ok)


BUF = np.zeros(64 * 64 * 3, np.uint8)
P = BUF.ctypes.data

FRAME_CASES = [   # (frames, w, h, nimg, message)
    ([P], [8], [8], 0, "nimg 0 outside 1..2"),
    ([P, P, P], [8] * 3, [8] * 3, 3, "nimg 3 outside 1..2"),
    (None, [8], [8], 1, "null frames array"),
    ([P], None, [8], 1, "null w / h array"),
    ([P], [8], None, 1, "null w / h array"),
    ([P, None], [8, 8], [8, 8], 2, "frame 1 is null"),
    ([P], [0], [8], 1, "frame 0 has size 0x8"),
    ([P], [8], [-3], 1, "frame 0 has size 8x-3"),
    ([P, P], [8, 40000], [8, 20000], 2, "frame 1 has more than INT_MAX bytes"),
]


@pytest.mark.parametrize("which", ["predict", "submit"])
@pytest.mark.parametrize("case", range(len(FRAME_CASES)))
def test_frame_calls_reject_bad_arguments(net, which, case):
    import yolo2_light_b200 as yb
    frames, w, h, nimg, msg = FRAME_CASES[case]
    with pytest.raises(yb.YbError, match=msg.replace("..", r"\.\.")):
        _call(net, which, frames, w, h, nimg)


@pytest.mark.parametrize("which", ["detect", "submit"])
@pytest.mark.parametrize("max_rows", [0, -1, 16385])
def test_max_rows_out_of_range(net, which, max_rows):
    import yolo2_light_b200 as yb
    with pytest.raises(yb.YbError, match=r"max_rows must be in 1\.\.16384"):
        _call(net, which, [P], [8], [8], 1, max_rows=max_rows)


@pytest.mark.parametrize("w,h,nimg,msg", [([8], [8], 0, "nimg 0 outside"), ([8] * 3, [8] * 3, 3, "nimg 3 outside"),
                                          (None, [8], 1, "null w / h"), ([8], [0], 1, "frame 0 has size 8x0")])
def test_detect_frames_rejects_bad_sizes(net, w, h, nimg, msg):
    import yolo2_light_b200 as yb
    with pytest.raises(yb.YbError, match=msg):
        _call(net, "detect", None, w, h, nimg)


@pytest.mark.parametrize("frames,msg", [
    ([np.zeros((8, 8, 3), np.float32)], "frame 0 must be a uint8"),
    ([np.zeros((8, 8, 3), np.uint8), np.zeros((1, 8, 8, 3), np.uint8)], "frame 1 must be a uint8"),
    ([np.zeros((8, 8), np.uint8)], "frame 0 must be a uint8"),
    ([np.zeros((8, 8, 4), np.uint8)], "frame 0 must be a uint8"),
    ([[[[0, 0, 0]]]], "frame 0 must be a uint8"),
    ([], "0 frames, the network takes 1..2"),
    ([np.zeros((8, 8, 3), np.uint8)] * 3, "3 frames, the network takes 1..2"),
])
def test_python_mirror_rejects_bad_frames(net, frames, msg):
    import yolo2_light_b200 as yb
    with pytest.raises(yb.YbError, match=msg.replace("..", r"\.\.")):
        net.predict_frames_u8(frames)
    with pytest.raises(yb.YbError, match=msg.replace("..", r"\.\.")):
        net.submit_frames_u8(frames, 0.5)
